// Package csvplus — cgo binding of the H100 hot path behind the csvplus API names (maxim2266/csvplus).
//
// SOURCE ONLY: this image has no Go toolchain, so these files have never been compiled.  They are the Go layer
// INTEGRATION.md describes: the public names, signatures, panics and error texts of the reference, lowered to the C ABI
// of include/csvplus_b200.h.  The same ABI is exercised for real from Python (ctypes) and C++ (host/csvplus.hpp).
//
// abi.go: handles, string marshalling, error mapping.  Nothing in this package parses, filters, sorts or joins on
// the CPU; the only per-row Go code is what the reference also runs per row: opaque user closures and the final RowFunc.
package csvplus

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../csvplus_b200 -lcsvplus_b200
#include <stdlib.h>
#include <string.h>
#include "csvplus_b200.h"
*/
import "C"

import (
	"errors"
	"fmt"
	"runtime"
	"sync"
	"unsafe"
)

// DataSourceError keeps the reference's definition (csvplus.go:1230-1238).
type DataSourceError struct {
	Line uint64
	Err  error
}

// Error prints `row N: msg` like csvplus.go:1236-1238.
func (e *DataSourceError) Error() string { return fmt.Sprintf(`row %d: %s`, e.Line, e.Err) }

// Unwrap exposes the inner error to errors.Is / errors.As.
func (e *DataSourceError) Unwrap() error { return e.Err }

// Context is one device + one CUDA stream (cpb_ctx).  A context serialises its calls; goroutines that need
// concurrency use one context each (NewContext).
type Context struct {
	h *C.cpb_ctx
}

var (
	defaultCtx  *Context
	defaultOnce sync.Once
)

// NewContext creates a context on the given CUDA device.  There is no CPU fallback: without a usable sm_90a
// (H100) device this fails.
func NewContext(device int) (*Context, error) {
	var h *C.cpb_ctx
	if st := C.cpb_init(C.int(device), &h); st != C.CPB_OK {
		return nil, fmt.Errorf("csvplus: cpb_init(device %d) failed with status %d (there is no CPU fallback)", device, int(st))
	}
	c := &Context{h}
	runtime.SetFinalizer(c, func(c *Context) { c.Close() })
	return c, nil
}

// Reserve maps nbytes of device memory into the context's pool ahead of time (cpb_pool_reserve), so that a steady loop
// of parses and joins never waits for the driver to map pages.  Optional.
func (c *Context) Reserve(nbytes uint64) error {
	if st := C.cpb_pool_reserve(c.h, C.uint64_t(nbytes)); st != C.CPB_OK {
		return fmt.Errorf("csvplus: cpb_pool_reserve(%d) failed with status %d", nbytes, int(st))
	}
	return nil
}

// Close releases the context; tables and indices created by it must be closed first.
func (c *Context) Close() {
	if c.h != nil {
		C.cpb_shutdown(c.h)
		c.h = nil
	}
}

func ctx() *Context {
	defaultOnce.Do(func() {
		c, err := NewContext(0)
		if err != nil {
			panic(err.Error())
		}
		defaultCtx = c
	})
	return defaultCtx
}

// InitMulti creates one context per device sharing one NCCL communicator (cpb_init_multi, SURVEY §8e).
func InitMulti(devices []int) ([]*Context, error) {
	if len(devices) == 0 {
		return nil, errors.New("csvplus: InitMulti needs at least one device")
	}
	devs := make([]C.int, len(devices))
	for i, d := range devices {
		devs[i] = C.int(d)
	}
	hs := make([]*C.cpb_ctx, len(devices))
	if st := C.cpb_init_multi(&devs[0], C.int(len(devs)), &hs[0]); st != C.CPB_OK {
		return nil, fmt.Errorf("csvplus: cpb_init_multi failed with status %d", int(st))
	}
	out := make([]*Context, len(hs))
	for i, h := range hs {
		out[i] = &Context{h}
	}
	return out, nil
}

// cstrs marshals Go strings into a C array of cpb_str; free() releases the C copies.
type cstrs struct {
	arr  []C.cpb_str
	keep []unsafe.Pointer
}

func newCstrs(items []string) *cstrs {
	s := &cstrs{arr: make([]C.cpb_str, len(items)+1)}
	for i, it := range items {
		p := C.CString(it)
		s.keep = append(s.keep, unsafe.Pointer(p))
		s.arr[i] = C.cpb_str{ptr: p, len: C.uint64_t(len(it))}
	}
	return s
}

func (s *cstrs) ptr() *C.cpb_str { return &s.arr[0] }

func (s *cstrs) free() {
	for _, p := range s.keep {
		C.free(p)
	}
	s.keep = nil
}

// mapErr turns (status, cpb_error) into the reference's error values: DataSourceError{Line, Err} when the
// reference wraps the message as `row N: ...` (csvplus.go:1209-1227, :243), a plain error otherwise.
func mapErr(st C.int, e *C.cpb_error) error {
	if st == C.CPB_OK {
		return nil
	}
	msg := C.GoString(&e.msg[0])
	if msg == "" {
		msg = fmt.Sprintf("csvplus: call failed with status %d", int(st))
	}
	if st == C.CPB_ERR_DATA && e.has_line != 0 {
		return &DataSourceError{Line: uint64(e.line), Err: errors.New(msg)}
	}
	return errors.New(msg)
}

// Table wraps cpb_table: a columnar batch of rows in HBM.
type Table struct {
	c *Context
	h *C.cpb_table
}

func newTable(c *Context, h *C.cpb_table) *Table {
	t := &Table{c, h}
	runtime.SetFinalizer(t, func(t *Table) { t.Close() })
	return t
}

// Close releases the device memory of the table.
func (t *Table) Close() {
	if t.h != nil {
		C.cpb_table_free(t.h)
		t.h = nil
	}
}

// NumRows returns the number of rows.
func (t *Table) NumRows() int64 { return int64(C.cpb_table_num_rows(t.h)) }

// Columns returns the column names.
func (t *Table) Columns() []string {
	n := int(C.cpb_table_num_cols(t.h))
	out := make([]string, n)
	for i := 0; i < n; i++ {
		var nm C.cpb_str
		C.cpb_table_col_name(t.h, C.int(i), &nm)
		out[i] = C.GoStringN(nm.ptr, C.int(nm.len))
	}
	return out
}

// rows materialises rows [lo, hi) as []Row: the boundary where opaque Go closures and the final RowFunc run.
func (t *Table) rows(lo, hi int64) ([]Row, error) {
	if hi > t.NumRows() {
		hi = t.NumRows()
	}
	if hi <= lo {
		return nil, nil
	}
	names := t.Columns()
	out := make([]Row, hi-lo)
	for i := range out {
		out[i] = make(Row, len(names))
	}
	for ci, name := range names {
		var nb C.uint64_t
		if st := C.cpb_table_col_bytes(t.c.h, t.h, C.int(ci), C.int64_t(lo), C.int64_t(hi), &nb); st != C.CPB_OK {
			return nil, fmt.Errorf("csvplus: cpb_table_col_bytes failed with status %d", int(st))
		}
		off := make([]int64, hi-lo+1)
		data := make([]byte, uint64(nb)+1)
		if st := C.cpb_table_fetch_column(t.c.h, t.h, C.int(ci), C.int64_t(lo), C.int64_t(hi), (*C.int64_t)(unsafe.Pointer(&off[0])),
			(*C.uint8_t)(unsafe.Pointer(&data[0])), C.uint64_t(len(data))); st != C.CPB_OK {
			return nil, fmt.Errorf("csvplus: cpb_table_fetch_column failed with status %d", int(st))
		}
		for i := range out {
			out[i][name] = string(data[off[i]:off[i+1]])
		}
	}
	return out, nil
}

// tableFromRows uploads rows that share one column set (TakeRows semantics, cpb_table_from_host).
func tableFromRows(c *Context, rows []Row) (*Table, error) {
	var names []string
	if len(rows) > 0 {
		names = rows[0].Header()
	}
	for _, r := range rows {
		if len(r) != len(names) {
			return nil, errors.New("csvplus: rows with different column sets cannot be uploaded as one table")
		}
	}
	cn := newCstrs(names)
	defer cn.free()
	offs := make([][]int64, len(names))
	datas := make([][]byte, len(names))
	offp := make([]*C.int64_t, len(names)+1)
	datp := make([]*C.uint8_t, len(names)+1)
	for k, name := range names {
		off := make([]int64, len(rows)+1)
		var buf []byte
		for i, r := range rows {
			v, found := r[name]
			if !found {
				return nil, errors.New("csvplus: rows with different column sets cannot be uploaded as one table")
			}
			buf = append(buf, v...)
			off[i+1] = int64(len(buf))
		}
		buf = append(buf, 0)
		offs[k], datas[k] = off, buf
	}
	// the pointer arrays live in C memory for the duration of the call (cgo: no Go pointers to Go pointers)
	po := (**C.int64_t)(C.malloc(C.size_t(len(names)+1) * C.size_t(unsafe.Sizeof(offp[0]))))
	pd := (**C.uint8_t)(C.malloc(C.size_t(len(names)+1) * C.size_t(unsafe.Sizeof(datp[0]))))
	defer C.free(unsafe.Pointer(po))
	defer C.free(unsafe.Pointer(pd))
	var pins runtime.Pinner
	defer pins.Unpin()
	poS := unsafe.Slice(po, len(names)+1)
	pdS := unsafe.Slice(pd, len(names)+1)
	for k := range names {
		pins.Pin(&offs[k][0])
		pins.Pin(&datas[k][0])
		poS[k] = (*C.int64_t)(unsafe.Pointer(&offs[k][0]))
		pdS[k] = (*C.uint8_t)(unsafe.Pointer(&datas[k][0]))
	}
	var h *C.cpb_table
	if st := C.cpb_table_from_host(c.h, C.int(len(names)), cn.ptr(), po, pd, C.int64_t(len(rows)), &h); st != C.CPB_OK {
		return nil, fmt.Errorf("csvplus: cpb_table_from_host failed with status %d", int(st))
	}
	return newTable(c, h), nil
}
