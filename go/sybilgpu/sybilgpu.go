// Package sybilgpu is the cgo shim a sybil maintainer adds to run
// Table.LoadAndQueryRecords (src/lib/table_query.go:18) on libsybilgpu.so.
//
// NOT COMPILED IN THIS REPOSITORY'S BUILD IMAGE (no Go toolchain there); it is
// written against include/sybilgpu.h and mirrors, call for call, what
// sybil_b200/engine.py does through ctypes (which IS exercised by the tests).
//
// Division of labour (INTEGRATION.md): Go keeps block enumeration, gob decoding
// (file_decoder.go:27-81), QuerySpec construction, regexp evaluation and
// printing; the library does staging, decode, filter, group-by, histograms,
// CombineResults and sorting.
package sybilgpu

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../sybil_b200/csrc -lsybilgpu -Wl,-rpath,${SRCDIR}/../../sybil_b200/csrc
#include <stdlib.h>
#include "sybilgpu.h"
*/
import "C"

import (
	"errors"
	"runtime"
	"unsafe"
)

// Ctx wraps sg_ctx: one per process and GPU.
type Ctx struct{ h *C.sg_ctx }

func Create(device int) (*Ctx, error) {
	var st C.int
	h := C.sg_create(C.int(device), &st)
	if st != C.SG_OK {
		msg := C.GoString(C.sg_last_error(h))
		C.sg_destroy(h)
		return nil, errors.New("sybilgpu: " + msg)
	}
	return &Ctx{h}, nil
}

func (c *Ctx) err() error { return errors.New("sybilgpu: " + C.GoString(C.sg_last_error(c.h))) }
func (c *Ctx) Close()     { C.sg_destroy(c.h) }

// Pinned returns cudaHostAlloc'd memory as a byte slice; gob-decode column
// arrays into slices carved from it so staging DMAs without a bounce copy.
func (c *Ctx) Pinned(n int) []byte {
	p := C.sg_pinned_alloc(c.h, C.size_t(n))
	if p == nil {
		return nil
	}
	return unsafe.Slice((*byte)(p), n)
}

// Table wraps sg_table: blocks staged once into HBM.
type Table struct {
	c *Ctx
	h *C.sg_table
}

// NewTable takes the (shortened) key table's column types: sybil.KeyTypes
// (INT_VAL = 1, STR_VAL = 2, record.go:14-19).
func (c *Ctx) NewTable(colTypes []int32) (*Table, error) {
	h := C.sg_table_create(c.h, C.int32_t(len(colTypes)), (*C.int32_t)(unsafe.Pointer(&colTypes[0])))
	if h == nil {
		return nil, c.err()
	}
	return &Table{c, h}, nil
}

// IntColumn / StrColumn are the decoded SavedIntColumn / SavedStrColumn
// (column_store.go:46-64) with Bins flattened: BinOffsets[i]..BinOffsets[i+1]
// delimit Bins[i].Records inside RecordIDs.
type Column struct {
	Slot        int32
	IsStr       bool
	// IsSet: a SavedSetColumn (column_store.go:66-74, ABI v4).  Handed over in the bucket form only (BinValues =
	// tag ids of StringTable, a row may sit in several bins); a file in the non-bucketed form (Values [][]int32) is
	// turned into bins by the caller, len(Values) goes into SetNumValues (sybilgpu.h).
	IsSet        bool
	SetNumValues uint32
	BucketEnc   bool // BucketEncoded
	DeltaIDs    bool // DeltaEncodedIDs
	DeltaValues bool // ValueEncoded
	BinValues   []int64
	BinOffsets  []uint32
	RecordIDs   []uint32
	ValuesI64   []int64
	ValuesI32   []int32
	// Narrow forms (ABI v3, sg_column_desc.id_bits / value_bits): a decoder that keeps gob's varints narrow
	// fills these INSTEAD of the wide slices above; 2-4x fewer bytes cross PCIe and sit in HBM.
	RecordIDs16 []uint16 // bucket columns: ids / gaps (always < 65,536 in a valid block)
	Deltas32    []int32  // int value arrays, ValueEncoded: value k = ValueBase + Deltas[0] + ... + Deltas[k]
	Deltas16    []int16  //   (the same, 16-bit)
	ValueBase   int64
	Values16    []uint16 // str value arrays: local string ids
	DictBytes   []byte   // StringTable concatenated
	DictOffsets []uint32 // len(StringTable)+1
}

type IntInfo struct {
	Slot     int32
	Min, Max int64
}

// pin makes a Go slice's backing array safe to store in C memory for the duration of the call (cgo pointer
// rules): runtime.Pinner keeps the collector from moving it.  Slices carved from Ctx.Pinned are C memory
// already and pinning them is a no-op.
func pin[T any](p *runtime.Pinner, s []T) unsafe.Pointer {
	if len(s) == 0 {
		return nil
	}
	d := unsafe.SliceData(s)
	p.Pin(d)
	return unsafe.Pointer(d)
}

// AddBlock stages one block (LoadBlockFromDir + unpack*Col, table_block_io.go:225-310).
// Small arrays (bin values, offsets, string tables) are read during the call; the big ones (record ids,
// values) are DMA'd asynchronously when they lie in memory from Ctx.Pinned and must stay untouched until
// Table.Sync returns (INTEGRATION.md §3) — Go-allocated slices are copied through the library's own staging
// before the call returns.  UNTESTED: this file has never been compiled (no Go toolchain in the build image).
func (t *Table) AddBlock(index int64, numRecords int32, cols []Column, info []IntInfo) error {
	var pinner runtime.Pinner
	defer pinner.Unpin()
	cdesc := (*C.sg_column_desc)(C.calloc(C.size_t(len(cols)+1), C.size_t(unsafe.Sizeof(C.sg_column_desc{}))))
	defer C.free(unsafe.Pointer(cdesc))
	cs := unsafe.Slice(cdesc, len(cols)+1)
	for i, col := range cols {
		d := &cs[i]
		d.col_slot = C.int32_t(col.Slot)
		d.col_type = C.SG_COL_INT
		if col.IsStr {
			d.col_type = C.SG_COL_STR
		}
		if col.IsSet {
			d.col_type = C.SG_COL_SET
		}
		if col.BucketEnc {
			d.encoding = C.SG_ENC_BUCKET
			d.nbins = C.uint32_t(len(col.BinValues))
			d.nrecord_ids = C.uint32_t(len(col.RecordIDs))
			d.bin_values = (*C.int64_t)(pin(&pinner, col.BinValues))
			d.bin_offsets = (*C.uint32_t)(pin(&pinner, col.BinOffsets))
			if len(col.RecordIDs16) > 0 {
				d.nrecord_ids = C.uint32_t(len(col.RecordIDs16))
				d.record_ids = (*C.uint32_t)(pin(&pinner, col.RecordIDs16))
				d.id_bits = 16
			} else {
				d.record_ids = (*C.uint32_t)(pin(&pinner, col.RecordIDs))
			}
		} else {
			d.encoding = C.SG_ENC_VALUES
			switch {
			case col.IsStr && len(col.Values16) > 0:
				d.nvalues = C.uint32_t(len(col.Values16))
				d.values_i32 = (*C.int32_t)(pin(&pinner, col.Values16))
				d.value_bits = 16
			case col.IsStr:
				d.nvalues = C.uint32_t(len(col.ValuesI32))
				d.values_i32 = (*C.int32_t)(pin(&pinner, col.ValuesI32))
			case len(col.Deltas16) > 0:
				d.nvalues = C.uint32_t(len(col.Deltas16))
				d.values_i64 = (*C.int64_t)(pin(&pinner, col.Deltas16))
				d.value_bits, d.value_base = 16, C.int64_t(col.ValueBase)
			case len(col.Deltas32) > 0:
				d.nvalues = C.uint32_t(len(col.Deltas32))
				d.values_i64 = (*C.int64_t)(pin(&pinner, col.Deltas32))
				d.value_bits, d.value_base = 32, C.int64_t(col.ValueBase)
			default:
				d.nvalues = C.uint32_t(len(col.ValuesI64))
				d.values_i64 = (*C.int64_t)(pin(&pinner, col.ValuesI64))
			}
		}
		if col.DeltaIDs {
			d.delta_ids = 1
		}
		if col.DeltaValues {
			d.delta_values = 1
		}
		if col.IsSet {
			d.nvalues = C.uint32_t(col.SetNumValues)
		}
		if col.IsStr || col.IsSet {
			d.ndict = C.uint32_t(len(col.DictOffsets) - 1)
			d.dict_bytes = (*C.char)(pin(&pinner, col.DictBytes))
			d.dict_offsets = (*C.uint32_t)(pin(&pinner, col.DictOffsets))
		}
	}
	cinfo := (*C.sg_int_info)(C.calloc(C.size_t(len(info)+1), C.size_t(unsafe.Sizeof(C.sg_int_info{}))))
	defer C.free(unsafe.Pointer(cinfo))
	is := unsafe.Slice(cinfo, len(info)+1)
	for i, ii := range info {
		is[i].col_slot, is[i].min, is[i].max = C.int32_t(ii.Slot), C.int64_t(ii.Min), C.int64_t(ii.Max)
	}
	var b C.sg_block_desc
	b.block_index, b.num_records = C.int64_t(index), C.int32_t(numRecords)
	b.ncols, b.cols = C.int32_t(len(cols)), cdesc
	b.ninfo, b.info = C.int32_t(len(info)), cinfo
	if C.sg_table_add_block(t.h, &b) != C.SG_OK {
		return t.c.err()
	}
	return nil
}

// Query mirrors QueryParams (query_spec.go:25-41) plus the FLAGS/OPTS globals
// the hot path reads (config.go:30-121).
type Filter struct {
	Slot   int32
	IsStr  bool
	IsSet  bool  // SetFilter (filter.go:162-169): Op is SG_OP_IN / SG_OP_NIN, StrVal the tag
	Op     int32 // SG_OP_*
	IntVal int64
	StrVal string
	// for SG_OP_RE / SG_OP_NRE: regexp over the table's global dictionary, evaluated
	// by the caller (filter.go:215-237) into a bitset
	Lut []uint32
}
type Group struct {
	Slot  int32
	IsStr bool
}
type Agg struct {
	Slot             int32
	InfoMin, InfoMax int64 // Table.IntInfo[col] (table_column_info.go:18-24)
}
type Query struct {
	OpHist     bool // FLAGS.OP == "hist"
	LogHist    bool // FLAGS.LOG_HIST
	HistBucket int32
	Filters    []Filter
	Groups     []Group
	Aggs       []Agg
	TimeSlot   int32 // -1: none
	TimeBucket int64
	TimeMin    int64
	TimeMax    int64
	WeightSlot int32 // OPTS.WEIGHT_COL_ID, -1: unweighted (a zero-valued Query must set -1 explicitly)
	StrReplace []StrReplaced // OPTS.STR_REPLACEMENTS, one entry per rewritten str column

	// Rows without the weight column take the weight of the block's previous row that has it (1 if none), as
	// LoadAndQueryRecords does.  False: such a row fails the query with SG_ERR_UNSUPPORTED at finish.
	WeightCarry bool
	// A group-by whose accumulators would pass 24 GiB keeps accumulators for the groups that occur only, as sybil's
	// result map does (sg_query_set_sparse_groups).  False: such a query fails with SG_ERR_UNSUPPORTED.
	SparseGroups bool
	// Weighted and StrReplace group-bys whose keys go through the device hash table (or sparse group accumulators)
	// are folded on the device (sg_query_set_hashed_folds).  False: such a query fails with SG_ERR_UNSUPPORTED.
	HashedFolds bool
}

// StrReplaced carries, for one str column, the rewritten text of every string of its global dictionary
// (sg_table_dict_size / sg_table_dict_get order): Offsets has one more entry than there are strings.
type StrReplaced struct {
	Slot    int32
	Bytes   []byte
	Offsets []uint32
}

// Run is LoadAndQueryRecords for the staged blocks: returns the result handle.
// (Filling QuerySpec.Results from it is done by the caller with the sg_result_*
// accessors; see INTEGRATION.md for the field mapping.)
func (t *Table) Run(q *Query, allreduce bool) (*C.sg_result, error) {
	nf, ng, na := len(q.Filters), len(q.Groups), len(q.Aggs)
	fl := (*C.sg_filter_desc)(C.calloc(C.size_t(nf+1), C.size_t(unsafe.Sizeof(C.sg_filter_desc{}))))
	gr := (*C.sg_group_desc)(C.calloc(C.size_t(ng+1), C.size_t(unsafe.Sizeof(C.sg_group_desc{}))))
	ag := (*C.sg_agg_desc)(C.calloc(C.size_t(na+1), C.size_t(unsafe.Sizeof(C.sg_agg_desc{}))))
	defer C.free(unsafe.Pointer(fl))
	defer C.free(unsafe.Pointer(gr))
	defer C.free(unsafe.Pointer(ag))
	fs, gs, as := unsafe.Slice(fl, nf+1), unsafe.Slice(gr, ng+1), unsafe.Slice(ag, na+1)
	var cstrs []unsafe.Pointer
	for i, f := range q.Filters {
		fs[i].col_slot, fs[i].op, fs[i].int_value = C.int32_t(f.Slot), C.int32_t(f.Op), C.int64_t(f.IntVal)
		fs[i].col_type = C.SG_COL_INT
		if f.IsStr || f.IsSet {
			fs[i].col_type = C.SG_COL_STR
			if f.IsSet {
				fs[i].col_type = C.SG_COL_SET
			}
			p := C.CString(f.StrVal)
			cstrs = append(cstrs, unsafe.Pointer(p))
			fs[i].str_value, fs[i].str_len = p, C.int64_t(len(f.StrVal))
		}
	}
	defer func() {
		for _, p := range cstrs {
			C.free(p)
		}
	}()
	for i, g := range q.Groups {
		gs[i].col_slot, gs[i].col_type = C.int32_t(g.Slot), C.SG_COL_INT
		if g.IsStr {
			gs[i].col_type = C.SG_COL_STR
		}
	}
	for i, a := range q.Aggs {
		as[i].col_slot, as[i].info_min, as[i].info_max = C.int32_t(a.Slot), C.int64_t(a.InfoMin), C.int64_t(a.InfoMax)
	}
	var d C.sg_query_desc
	d.abi_version = C.SG_ABI_VERSION
	if q.OpHist {
		d.op_mode = C.SG_MODE_HIST
	}
	if q.LogHist {
		d.hist_kind = C.SG_HIST_MULTI
	}
	d.hist_bucket = C.int32_t(q.HistBucket)
	d.nfilters, d.ngroups, d.naggs = C.int32_t(nf), C.int32_t(ng), C.int32_t(na)
	d.filters, d.groups, d.aggs = fl, gr, ag
	d.time_col_slot, d.time_bucket = C.int32_t(q.TimeSlot), C.int64_t(q.TimeBucket)
	d.time_min, d.time_max = C.int64_t(q.TimeMin), C.int64_t(q.TimeMax)
	d.weight_col_slot = C.int32_t(q.WeightSlot) // -1: unweighted
	if q.WeightCarry { // rows without the column reuse the previous row's weight; else SG_ERR_UNSUPPORTED at finish
		d.weight_carry = 1
	}
	// SortResults(OrderBy, OrderAsc) and FLAGS.LIMIT (ABI v2)
	d.order_by_agg = C.SG_ORDER_COUNT
	if spec.OrderBy == "" {
		d.order_by_agg = C.SG_ORDER_NONE
	} else if spec.OrderBy != "$COUNT" {
		for i, a := range spec.Aggregations {
			if a.Name == spec.OrderBy {
				d.order_by_agg = C.int32_t(i)
			}
		}
	}
	if spec.OrderAsc {
		d.order_asc = 1
	}
	d.limit = C.int64_t(spec.Limit)
	h := C.sg_query_begin(t.c.h, t.h, &d)
	if h == nil {
		return nil, t.c.err()
	}
	defer C.sg_query_free(h)
	if q.SparseGroups && C.sg_query_set_sparse_groups(h, 1) != C.SG_OK {
		return nil, t.c.err()
	}
	if q.HashedFolds && C.sg_query_set_hashed_folds(h, 1) != C.SG_OK {
		return nil, t.c.err()
	}
	for i, f := range q.Filters {
		if f.Lut != nil {
			n := C.sg_table_dict_size(t.h, C.int32_t(f.Slot))
			if int64(len(f.Lut)) < (int64(n)+31)/32 { // one bit per global string id of the column
				return nil, errors.New("sybilgpu: regex LUT shorter than the column's dictionary")
			}
			if C.sg_query_set_str_lut(h, C.int32_t(i), (*C.uint32_t)(unsafe.Pointer(&f.Lut[0])), n) != C.SG_OK {
				return nil, t.c.err()
			}
		}
	}
	// StrReplace (table_query.go:34-50): the caller rewrote every string of the column's dictionary with
	// regexp.ReplaceAllString (and built the Luts of that column's filters on the rewritten strings)
	for _, sr := range q.StrReplace {
		var pinner runtime.Pinner
		rc := C.sg_query_set_str_replace(h, C.int32_t(sr.Slot), (*C.char)(pin(&pinner, sr.Bytes)),
			(*C.uint32_t)(pin(&pinner, sr.Offsets)), C.int64_t(len(sr.Offsets)-1))
		pinner.Unpin()
		if rc != C.SG_OK {
			return nil, t.c.err()
		}
	}
	if C.sg_query_run(h) != C.SG_OK {
		return nil, t.c.err()
	}
	if allreduce && C.sg_query_allreduce(h) != C.SG_OK {
		return nil, t.c.err()
	}
	var r *C.sg_result
	if C.sg_query_finish(h, &r) != C.SG_OK {
		return nil, t.c.err()
	}
	return r, nil
}
