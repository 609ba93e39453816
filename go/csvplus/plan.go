package csvplus

// plan.go: DataSource and its combinators (csvplus.go:207-608) as a lazily evaluated plan.
//
// DataSource keeps the reference's type — func(RowFunc) error — so user code calls it, stores it and defines methods'
// receivers exactly as before.  Every DataSource made by this package is a closure over a plan node.  A sink (calling
// the source with a RowFunc, ToRows, ToCsv, IndexOn, ...) lowers the recognisable prefix of the plan
//     parse -> SelectColumns/DropColumns -> Filter(Like/All/Any/Not) -> Join/Except -> Top/Drop ...
// to C-ABI calls and materialises Row maps only where an opaque closure or the final RowFunc needs them.
// How a combinator recognises its upstream: it calls the upstream DataSource with the package-private sentinel
// planProbe; sources of this package answer with their plan node (wrapped in an error value) instead of iterating.
// A foreign DataSource (a func the user wrote) is simply pulled by that call — exactly once, as the sink would —
// into host rows, and continues as a TakeRows source.

/*
#include <stdlib.h>
#include "csvplus_b200.h"
*/
import "C"

import (
	"bytes"
	"encoding/json"
	"errors"
	"io"
	"os"
	"reflect"
	"unsafe"
)

// DataSource is the iterator type of the library (csvplus.go:215).
type DataSource func(RowFunc) error

type opKind int

const (
	opParse opKind = iota // Take(reader)
	opRows                // TakeRows / a pulled foreign source
	opTable               // an Index or a device table
	opFilter
	opMap
	opTransform
	opValidate
	opTop
	opDrop
	opTakeWhile
	opDropWhile
	opDropColumns
	opSelectColumns
	opJoin
	opExcept
)

type plan struct {
	kind     opKind
	up       *plan
	reader   *Reader
	rows     []Row
	rowsErr  error // error a pulled foreign source ended with
	table    *Table
	lineBase uint64
	pred     func(Row) bool
	mapf     func(Row) Row
	trans    func(Row) (Row, error)
	valid    func(Row) error
	n        uint64
	columns  []string
	index    *Index
}

// ---- the probe protocol
var foreignRows []Row

func planProbe(row Row) error { // only ever called by foreign sources: collect what they deliver
	foreignRows = append(foreignRows, row)
	return nil
}

var planProbePC = reflect.ValueOf(planProbe).Pointer()

func isPlanProbe(fn RowFunc) bool { return reflect.ValueOf(fn).Pointer() == planProbePC }

type planReply struct{ node *plan }

func (*planReply) Error() string { return "csvplus: internal plan probe" }

func planOf(src DataSource) *plan {
	probeMu.Lock()
	defer probeMu.Unlock()
	foreignRows = nil
	err := src(planProbe)
	var reply *planReply
	if errors.As(err, &reply) {
		return reply.node
	}
	rows := foreignRows
	foreignRows = nil
	return &plan{kind: opRows, rows: rows, rowsErr: err}
}

func newSource(node *plan) DataSource {
	return func(fn RowFunc) error {
		if isPlanProbe(fn) {
			return &planReply{node}
		}
		return node.run(fn)
	}
}

func (src DataSource) with(node *plan) DataSource {
	node.up = planOf(src)
	return newSource(node)
}

// Take converts anything with an Iterate method to a DataSource (csvplus.go:252).  Readers and Indices of this package
// become plan sources; anything else is pulled through its Iterate method when a sink runs.
func Take(src interface{ Iterate(fn RowFunc) error }) DataSource {
	switch s := src.(type) {
	case *Reader:
		return newSource(&plan{kind: opParse, reader: s})
	case *Index:
		return newSource(&plan{kind: opTable, table: s.table(), lineBase: 0})
	}
	return src.Iterate
}

// TakeRows converts a slice of Rows to a DataSource (csvplus.go:218).
func TakeRows(rows []Row) DataSource { return newSource(&plan{kind: opRows, rows: rows}) }

// Transform is the most generic row operation (csvplus.go:261): an empty result drops the row, an error stops.
func (src DataSource) Transform(trans func(Row) (Row, error)) DataSource {
	return src.with(&plan{kind: opTransform, trans: trans})
}

// Filter passes the rows for which pred is true (csvplus.go:276).  Like/All/Any/Not predicates run inside the kernels.
func (src DataSource) Filter(pred func(Row) bool) DataSource { return src.with(&plan{kind: opFilter, pred: pred}) }

// Map applies mf to every row (csvplus.go:290); an opaque closure: it runs on the host.
func (src DataSource) Map(mf func(Row) Row) DataSource { return src.with(&plan{kind: opMap, mapf: mf}) }

// Validate stops at the first row for which vf returns an error (csvplus.go:300).
func (src DataSource) Validate(vf func(Row) error) DataSource { return src.with(&plan{kind: opValidate, valid: vf}) }

// Top passes the first n rows (csvplus.go:313).
func (src DataSource) Top(n uint64) DataSource { return src.with(&plan{kind: opTop, n: n}) }

// Drop ignores the first n rows (csvplus.go:329).
func (src DataSource) Drop(n uint64) DataSource { return src.with(&plan{kind: opDrop, n: n}) }

// TakeWhile stops at the first row for which pred is false (csvplus.go:346).
func (src DataSource) TakeWhile(pred func(Row) bool) DataSource { return src.with(&plan{kind: opTakeWhile, pred: pred}) }

// DropWhile ignores rows while pred is true (csvplus.go:361).
func (src DataSource) DropWhile(pred func(Row) bool) DataSource { return src.with(&plan{kind: opDropWhile, pred: pred}) }

// DropColumns removes the columns from every row (csvplus.go:493).
func (src DataSource) DropColumns(columns ...string) DataSource {
	if len(columns) == 0 {
		panic("no columns specified in DropColumns()")
	}
	return src.with(&plan{kind: opDropColumns, columns: columns})
}

// SelectColumns leaves only the named columns; a missing one is an error (csvplus.go:511).
func (src DataSource) SelectColumns(columns ...string) DataSource {
	if len(columns) == 0 {
		panic("no columns specified in SelectColumns()")
	}
	return src.with(&plan{kind: opSelectColumns, columns: columns})
}

// Join is the inner join of the source with the index (csvplus.go:545): no columns = the index's own columns.
func (src DataSource) Join(index *Index, columns ...string) DataSource {
	if len(columns) == 0 {
		columns = index.columns
	} else if len(columns) > len(index.columns) {
		panic("too many source columns in Join()")
	}
	return src.with(&plan{kind: opJoin, index: index, columns: columns})
}

// Except passes the rows that have no match in the index (csvplus.go:588).
func (src DataSource) Except(index *Index, columns ...string) DataSource {
	if len(columns) == 0 {
		columns = index.columns
	} else if len(columns) > len(index.columns) {
		panic("too many source columns in Except()")
	}
	return src.with(&plan{kind: opExcept, index: index, columns: columns})
}

// ---- evaluation

// result of evaluating a plan: a device table, or host rows (after an opaque closure), plus the error that ended
// the source after those rows (the reference delivers the rows before it, then returns it)
type result struct {
	table    *Table
	rows     []Row
	onHost   bool
	lineBase uint64 // DataSourceError.Line of row 0 for errors raised by host callbacks
	err      error
}

func (r *result) hostRows() ([]Row, error) {
	if r.onHost {
		return r.rows, nil
	}
	if r.table == nil {
		return nil, nil
	}
	return r.table.rows(0, r.table.NumRows())
}

func (r *result) deviceTable(c *Context) (*Table, error) {
	if !r.onHost {
		return r.table, nil
	}
	return tableFromRows(c, r.rows)
}

func (p *plan) context() *Context {
	for q := p; q != nil; q = q.up {
		if q.reader != nil {
			return q.reader.context()
		}
		if q.table != nil {
			return q.table.c
		}
	}
	return ctx()
}

func cNames(cols []string) *cstrs { return newCstrs(cols) }

func (p *plan) eval() *result {
	switch p.kind {
	case opParse:
		t, err := p.reader.parse(nil)
		base := uint64(1)
		if p.reader.headerFromFirstRow {
			base = 2
		}
		return &result{table: t, lineBase: base, err: err}
	case opRows:
		return &result{rows: p.rows, onHost: true, err: p.rowsErr}
	case opTable:
		return &result{table: p.table, lineBase: p.lineBase}
	}
	// a recognisable Filter directly on a Reader is fused into the scan kernel (rows failing it are never materialised)
	if p.kind == opFilter && p.up.kind == opParse {
		if spec := describe(p.pred); spec != nil {
			t, err := p.up.reader.parse(spec)
			base := uint64(1)
			if p.up.reader.headerFromFirstRow {
				base = 2
			}
			return &result{table: t, lineBase: base, err: err}
		}
	}
	in := p.up.eval()
	c := p.context()
	switch p.kind {
	case opFilter:
		if spec := describe(p.pred); spec != nil && !in.onHost && in.table != nil {
			cp := spec.toC()
			defer cp.free()
			var out *C.cpb_table
			if st := C.cpb_table_filter(c.h, in.table.h, cp.root, &out); st != C.CPB_OK {
				return &result{err: errors.New("csvplus: cpb_table_filter failed")}
			}
			return &result{table: newTable(c, out), lineBase: in.lineBase, err: in.err}
		}
	case opSelectColumns, opDropColumns:
		if !in.onHost && in.table != nil {
			cn := cNames(p.columns)
			defer cn.free()
			var out *C.cpb_table
			var e C.cpb_error
			var st C.int
			if p.kind == opSelectColumns {
				st = C.int(C.cpb_table_select(c.h, in.table.h, cn.ptr(), C.int(len(p.columns)), &out, &e))
			} else {
				st = C.int(C.cpb_table_drop(c.h, in.table.h, cn.ptr(), C.int(len(p.columns)), &out))
			}
			if st != C.CPB_OK {
				return &result{err: mapErr(st, &e)}
			}
			return &result{table: newTable(c, out), lineBase: in.lineBase, err: in.err}
		}
	case opTop, opDrop:
		if !in.onHost && in.table != nil {
			lo, hi := int64(0), in.table.NumRows()
			if p.kind == opTop {
				if int64(p.n) < hi {
					hi = int64(p.n)
					in.err = nil // the reference stops pulling (io.EOF) before it could meet the later error
				}
			} else {
				lo = int64(p.n)
			}
			var out *C.cpb_table
			if st := C.cpb_table_slice(c.h, in.table.h, C.int64_t(lo), C.int64_t(hi), &out); st != C.CPB_OK {
				return &result{err: errors.New("csvplus: cpb_table_slice failed")}
			}
			return &result{table: newTable(c, out), lineBase: in.lineBase + uint64(lo), err: in.err}
		}
	case opJoin, opExcept:
		probe, err := in.deviceTable(c)
		if err != nil {
			return &result{err: err}
		}
		if probe == nil {
			return &result{err: in.err}
		}
		cn := cNames(p.columns)
		defer cn.free()
		var out *C.cpb_table
		var e C.cpb_error
		var st C.int
		if p.kind == opJoin {
			st = C.int(C.cpb_join(c.h, probe.h, p.index.h, cn.ptr(), C.int(len(p.columns)), &out, &e))
		} else {
			st = C.int(C.cpb_except(c.h, probe.h, p.index.h, cn.ptr(), C.int(len(p.columns)), &out, &e))
		}
		if st != C.CPB_OK {
			return &result{err: mapErr(st, &e)}
		}
		return &result{table: newTable(c, out), lineBase: in.lineBase, err: in.err}
	}
	// everything else is an opaque closure (or a recognisable op after one): host rows, the reference's own semantics
	rows, err := in.hostRows()
	if err != nil {
		return &result{err: err}
	}
	out := make([]Row, 0, len(rows))
	wrap := func(i int, e error) error { // csvplus.go:1137 / :243: errors of downstream callbacks carry the row's line
		var dse *DataSourceError
		if errors.As(e, &dse) {
			return e
		}
		return &DataSourceError{Line: in.lineBase + uint64(i), Err: e}
	}
	stopped := false
	yield := false
	counter := p.n
	var failed error
loop:
	for i, row := range rows {
		switch p.kind {
		case opFilter:
			if p.pred(row) {
				out = append(out, row)
			}
		case opMap:
			out = append(out, p.mapf(row))
		case opTransform:
			nr, e := p.trans(row)
			if e != nil {
				failed = wrap(i, e)
				break loop
			}
			if len(nr) > 0 {
				out = append(out, nr)
			}
		case opValidate:
			if e := p.valid(row); e != nil {
				failed = wrap(i, e)
				break loop
			}
			out = append(out, row)
		case opTop:
			if counter == 0 {
				stopped = true
				break loop
			}
			counter--
			out = append(out, row)
		case opDrop:
			if counter == 0 {
				out = append(out, row)
			} else {
				counter--
			}
		case opTakeWhile:
			if !p.pred(row) {
				stopped = true
				break loop
			}
			out = append(out, row)
		case opDropWhile:
			if yield = yield || !p.pred(row); yield {
				out = append(out, row)
			}
		case opDropColumns:
			for _, col := range p.columns {
				delete(row, col)
			}
			out = append(out, row)
		case opSelectColumns:
			nr, e := row.Select(p.columns...)
			if e != nil {
				failed = wrap(i, e)
				break loop
			}
			out = append(out, nr)
		}
	}
	res := &result{rows: out, onHost: true, lineBase: in.lineBase}
	switch {
	case failed != nil:
		res.err = failed
	case stopped:
		res.err = nil // io.EOF upstream: the source is not pulled any further
	default:
		res.err = in.err
	}
	return res
}

// run is the final sink: evaluate, hand every row to fn, then return the error the source ended with.
func (p *plan) run(fn RowFunc) error {
	res := p.eval()
	rows, err := res.hostRows()
	if err != nil {
		return err
	}
	for i, row := range rows {
		if e := fn(row); e != nil {
			if e == io.EOF {
				return nil
			}
			var dse *DataSourceError
			if errors.As(e, &dse) {
				return e
			}
			return &DataSourceError{Line: res.lineBase + uint64(i), Err: e}
		}
	}
	return res.err
}

// ---- sinks

// ToRows pulls the source into a slice (csvplus.go:483).
func (src DataSource) ToRows() (rows []Row, err error) {
	err = src(func(row Row) error {
		rows = append(rows, row)
		return nil
	})
	return
}

// ToCsv writes the selected columns in canonical .csv form (csvplus.go:379).  A device-resident result is serialised
// by the GPU (cpb_table_to_csv); host rows go through the same kernel after an upload.
func (src DataSource) ToCsv(out io.Writer, columns ...string) error {
	if len(columns) == 0 {
		panic("empty column list in ToCsv() function")
	}
	p := planOf(src)
	res := p.eval()
	c := p.context()
	t, err := res.deviceTable(c)
	if err != nil {
		return err
	}
	if t == nil {
		if res.err != nil {
			return res.err
		}
		var e error
		t, e = tableFromRows(c, nil)
		if e != nil {
			return e
		}
	}
	cn := cNames(columns)
	defer cn.free()
	var buf unsafe.Pointer
	var n C.uint64_t
	var e C.cpb_error
	if st := C.cpb_table_to_csv(c.h, t.h, cn.ptr(), C.int(len(columns)), &buf, &n, &e); st != C.CPB_OK {
		return mapErr(C.int(st), &e)
	}
	defer C.cpb_host_free(c.h, buf)
	if n > 0 {
		if _, werr := out.Write(unsafe.Slice((*byte)(buf), int(n))); werr != nil {
			return werr
		}
	}
	return res.err
}

// writeFile creates the file, runs fn on it and removes the file again on error or panic (csvplus.go:417-443).
func writeFile(name string, fn func(io.Writer) error) (err error) {
	file, err := os.Create(name)
	if err != nil {
		return err
	}
	defer func() {
		if p := recover(); p != nil {
			file.Close()
			os.Remove(name)
			panic(p)
		}
		if e := file.Close(); e != nil && err == nil {
			err = e
		}
		if err != nil {
			os.Remove(name)
		}
	}()
	return fn(file)
}

// ToCsvFile is ToCsv into a file; the file is removed on error (csvplus.go:411).
func (src DataSource) ToCsvFile(name string, columns ...string) error {
	return writeFile(name, func(w io.Writer) error { return src.ToCsv(w, columns...) })
}

// jsonBatchRows is the number of rows per cpb_table_to_json_into call: one call produces less than 4 GiB.
const jsonBatchRows = 1 << 24

// ToJSON writes all rows as a JSON array of objects, one object per line (csvplus.go:446-474: json.Encoder with
// SetEscapeHTML(false), a comma before every element but the first).  A device-resident result is serialised by the
// GPU in row-range batches (cpb_table_to_json_into) through one reused pinned buffer; host rows (after an opaque
// closure) go through encoding/json.  When the source fails after some rows, out receives what the reference would
// have flushed before the error, and no closing ']'.
func (src DataSource) ToJSON(out io.Writer) error {
	p := planOf(src)
	res := p.eval()
	if res.onHost {
		return rowsToJSON(out, res.rows, res.err)
	}
	c := p.context()
	if res.table == nil {
		if res.err != nil {
			return res.err
		}
		_, err := out.Write([]byte("[]"))
		return err
	}
	n := res.table.NumRows()
	var buf unsafe.Pointer
	var capacity C.uint64_t
	defer func() {
		if buf != nil {
			C.cpb_host_free(c.h, buf)
		}
	}()
	var pending []byte
	for lo := int64(0); ; {
		hi := lo + jsonBatchRows
		if hi > n {
			hi = n
		}
		var part *C.cpb_table
		if st := C.cpb_table_slice(c.h, res.table.h, C.int64_t(lo), C.int64_t(hi), &part); st != C.CPB_OK {
			return errors.New("csvplus: cpb_table_slice failed")
		}
		first, last := C.int(0), C.int(0)
		if lo == 0 {
			first = 1
		}
		if hi == n && res.err == nil {
			last = 1
		}
		var w C.uint64_t
		var e C.cpb_error
		st := C.cpb_table_to_json_into(c.h, part, first, last, buf, capacity, &w, &e)
		C.cpb_table_free(part)
		if st == C.CPB_ERR_ARG && w > capacity { // grow the buffer to the size the batch needs and repeat it
			if buf != nil {
				C.cpb_host_free(c.h, buf)
				buf, capacity = nil, 0
			}
			if C.cpb_host_alloc(c.h, w+w/4, &buf) != C.CPB_OK {
				return errors.New("csvplus: cpb_host_alloc failed")
			}
			capacity = w + w/4
			continue
		}
		if st != C.CPB_OK {
			return mapErr(C.int(st), &e)
		}
		chunk := unsafe.Slice((*byte)(buf), int(w))
		if res.err == nil {
			if _, err := out.Write(chunk); err != nil {
				return err
			}
		} else {
			var err error
			if pending, err = writeFlushed(out, pending, chunk); err != nil {
				return err
			}
		}
		if lo = hi; lo >= n {
			break
		}
	}
	return res.err
}

// writeFlushed writes what the reference flushes of these rows when the source fails after them: its buffer goes out
// after every row that leaves more than 10 000 bytes pending.  A raw '\n' only ever ends a row, because the encoder
// escapes every newline inside a string.  Returns the bytes still pending.
func writeFlushed(out io.Writer, pending, chunk []byte) ([]byte, error) {
	for len(chunk) > 0 {
		i := bytes.IndexByte(chunk, '\n')
		if i < 0 {
			return append(pending, chunk...), nil
		}
		pending = append(pending, chunk[:i+1]...)
		chunk = chunk[i+1:]
		if len(pending) > 10000 {
			if _, err := out.Write(pending); err != nil {
				return nil, err
			}
			pending = pending[:0]
		}
	}
	return pending, nil
}

// rowsToJSON is the reference's ToJSON over rows left on the host, ended by srcErr.
func rowsToJSON(out io.Writer, rows []Row, srcErr error) error {
	var buff bytes.Buffer
	buff.WriteByte('[')
	enc := json.NewEncoder(&buff)
	enc.SetIndent("", "")
	enc.SetEscapeHTML(false)
	for i, row := range rows {
		if i > 0 {
			buff.WriteByte(',')
		}
		if e := enc.Encode(row); e != nil {
			return e
		}
		if buff.Len() > 10000 {
			if _, e := buff.WriteTo(out); e != nil {
				return e
			}
		}
	}
	if srcErr != nil {
		return srcErr
	}
	buff.WriteByte(']')
	_, err := buff.WriteTo(out)
	return err
}

// ToJSONFile is ToJSON into a file (csvplus.go:477).
func (src DataSource) ToJSONFile(name string) error { return writeFile(name, src.ToJSON) }
