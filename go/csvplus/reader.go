package csvplus

// reader.go: the Reader and its options (csvplus.go:922-1076) lowered to cpb_stream_* (cpb_parse_csv-compatible batches).

/*
#include <stdlib.h>
#include "csvplus_b200.h"
*/
import "C"

import (
	"bytes"
	"errors"
	"io"
	"os"
	"runtime"
	"unsafe"
)

type sourceFn func() (io.ReadCloser, error)

// StreamBatchBytes is the size of one piece of input pushed to the GPU (cpb_stream_push): the input is parsed in
// batches of whole records and never held whole in host memory.
var StreamBatchBytes = 128 << 20

// Reader is an iterable csv reader.  Its options have the reference's names and panics; Iterate reads the input in
// pieces of StreamBatchBytes, parses them on the GPU in batches of whole records (cpb_stream_*) and then hands the rows
// to the callback.
type Reader struct {
	source                       sourceFn
	delimiter, comment           rune
	numFields                    int
	lazyQuotes, trimLeadingSpace bool
	header                       map[string]int
	headerFromFirstRow           bool
	ctx                          *Context
}

func makeReader(src sourceFn) *Reader {
	return &Reader{source: src, delimiter: ',', headerFromFirstRow: true}
}

// FromFile binds a reader to a file; the file is opened on every iteration, so the source is re-iterable
// (csvplus.go:950-959).
func FromFile(name string) *Reader {
	return makeReader(func() (io.ReadCloser, error) { return os.Open(name) })
}

// FromReader constructs a reader over an io.Reader (one shot, csvplus.go:936).
func FromReader(input io.Reader) *Reader {
	return makeReader(func() (io.ReadCloser, error) { return io.NopCloser(input), nil })
}

// FromReadCloser is FromReader that also closes the input when the iteration ends (csvplus.go:943).
func FromReadCloser(input io.ReadCloser) *Reader {
	return makeReader(func() (io.ReadCloser, error) { return input, nil })
}

// OnContext makes the reader parse on the given context instead of the default one (not in the reference).
func (r *Reader) OnContext(c *Context) *Reader { r.ctx = c; return r }

// Delimiter sets the field delimiter.
func (r *Reader) Delimiter(c rune) *Reader { r.delimiter = c; return r }

// CommentChar sets the symbol that starts a comment line.
func (r *Reader) CommentChar(c rune) *Reader { r.comment = c; return r }

// LazyQuotes relaxes quote handling like encoding/csv's LazyQuotes.
func (r *Reader) LazyQuotes() *Reader { r.lazyQuotes = true; return r }

// TrimLeadingSpace ignores leading white space of every field.
func (r *Reader) TrimLeadingSpace() *Reader { r.trimLeadingSpace = true; return r }

// AssumeHeader names the columns of an input without a header row (csvplus.go:998-1012).
func (r *Reader) AssumeHeader(spec map[string]int) *Reader {
	if len(spec) == 0 {
		panic("Empty header spec")
	}
	for name, col := range spec {
		if col < 0 {
			panic("header spec: negative index for column " + name)
		}
	}
	r.header = spec
	r.headerFromFirstRow = false
	return r
}

// ExpectHeader verifies the first row against the specification; a negative index means "find by name"
// (csvplus.go:1020-1033).
func (r *Reader) ExpectHeader(spec map[string]int) *Reader {
	if len(spec) == 0 {
		panic("empty header spec")
	}
	r.header = make(map[string]int, len(spec))
	for name, col := range spec {
		r.header[name] = col
	}
	r.headerFromFirstRow = true
	return r
}

// SelectColumns names the columns to read; they are located in the first row (csvplus.go:1039-1056).
func (r *Reader) SelectColumns(names ...string) *Reader {
	if len(names) == 0 {
		panic("empty header spec")
	}
	r.header = make(map[string]int, len(names))
	for _, name := range names {
		if _, dup := r.header[name]; dup {
			panic("header spec: duplicate column name: " + name)
		}
		r.header[name] = -1
	}
	r.headerFromFirstRow = true
	return r
}

// NumFields sets the exact number of fields every record must have.
func (r *Reader) NumFields(n int) *Reader { r.numFields = n; return r }

// NumFieldsAuto: every record must have as many fields as the first one.
func (r *Reader) NumFieldsAuto() *Reader { return r.NumFields(0) }

// NumFieldsAny: records may have any number of fields; short ones are padded with empty values.
func (r *Reader) NumFieldsAny() *Reader { return r.NumFields(-1) }

func (r *Reader) context() *Context {
	if r.ctx != nil {
		return r.ctx
	}
	return ctx()
}

// parse lowers Reader.Iterate (+ an optional recognised predicate that directly follows it) to cpb_parse_csv when the
// input fits one batch, else to cpb_stream_*: the input is pushed in pinned pieces of StreamBatchBytes, each push parses the complete records received so far, and the batches'
// tables are concatenated (cpb_table_concat).  On a data error the table holds the rows the streaming reference would
// have delivered before failing.
func (r *Reader) parse(pred *predSpec) (*Table, error) {
	pathErr := func(err error) error { // csvplus.go:1216-1220: *os.PathError is reported as "op: err", everything is row 1
		var pe *os.PathError
		if errors.As(err, &pe) {
			return &DataSourceError{Line: 1, Err: errors.New(pe.Op + ": " + pe.Err.Error())}
		}
		return &DataSourceError{Line: 1, Err: err}
	}
	input, err := r.source()
	if err != nil {
		return nil, pathErr(err)
	}
	defer input.Close()
	// an input that fits one batch is parsed in one cpb_parse_csv call, staged at its own size
	first, err := io.ReadAll(io.LimitReader(input, int64(StreamBatchBytes)+1))
	if err != nil {
		return nil, pathErr(err)
	}
	opts := C.cpb_reader_opts{delimiter: C.uint32_t(r.delimiter), comment: C.uint32_t(r.comment), num_fields: C.int32_t(r.numFields)}
	if r.lazyQuotes {
		opts.lazy_quotes = 1
	}
	if r.trimLeadingSpace {
		opts.trim_leading_space = 1
	}
	if r.headerFromFirstRow {
		opts.header_from_first_row = 1
	}
	names := make([]string, 0, len(r.header))
	for name := range r.header {
		names = append(names, name)
	}
	cn := newCstrs(names)
	defer cn.free()
	spec := make([]C.cpb_header_col, len(names)+1)
	for i, name := range names {
		spec[i] = C.cpb_header_col{name: cn.arr[i], index: C.int32_t(r.header[name])}
	}
	var cpred *C.cpb_pred
	if pred != nil {
		cp := pred.toC()
		defer cp.free()
		cpred = cp.root
	}
	c := r.context()
	var e C.cpb_error
	if len(first) <= StreamBatchBytes {
		var staging unsafe.Pointer // pinned staging memory filled by the host, as INTEGRATION.md describes
		if len(first) > 0 {
			if s := C.cpb_host_alloc(c.h, C.uint64_t(len(first)), &staging); s != C.CPB_OK {
				return nil, errors.New("csvplus: cpb_host_alloc failed")
			}
			defer C.cpb_host_free(c.h, staging)
			C.memcpy(staging, unsafe.Pointer(&first[0]), C.size_t(len(first)))
		}
		var out *C.cpb_table
		s := C.cpb_parse_csv(c.h, staging, C.uint64_t(len(first)), 0, &opts, &spec[0], C.int(len(names)), cpred, &out, &e)
		var t *Table
		if out != nil {
			t = newTable(c, out)
		}
		return t, mapErr(C.int(s), &e)
	}
	src := io.MultiReader(bytes.NewReader(first), input)
	var st *C.cpb_stream
	if s := C.cpb_stream_open(c.h, &opts, &spec[0], C.int(len(names)), cpred, &st, &e); s != C.CPB_OK {
		return nil, mapErr(C.int(s), &e)
	}
	defer C.cpb_stream_free(st)
	// pinned staging memory filled by the host (io.ReadFull), as INTEGRATION.md describes; a piece stays untouched
	// until the cpb_stream_next after its push has returned
	var staging unsafe.Pointer
	if s := C.cpb_host_alloc(c.h, C.uint64_t(StreamBatchBytes), &staging); s != C.CPB_OK {
		return nil, errors.New("csvplus: cpb_host_alloc failed")
	}
	defer C.cpb_host_free(c.h, staging)
	buf := unsafe.Slice((*byte)(staging), StreamBatchBytes)
	var parts []*Table
	collect := func() (bool, error) { // one cpb_stream_next per push; false: the stream is done
		var out *C.cpb_table
		var done C.int
		s := C.cpb_stream_next(st, &out, &done, &e)
		if out != nil {
			parts = append(parts, newTable(c, out))
		}
		if s != C.CPB_OK {
			return false, mapErr(C.int(s), &e)
		}
		return done == 0, nil
	}
	var serr error
	for more := true; more; {
		n, rerr := io.ReadFull(src, buf)
		last := rerr == io.EOF || rerr == io.ErrUnexpectedEOF
		if rerr != nil && !last {
			return nil, pathErr(rerr)
		}
		if s := C.cpb_stream_push(st, staging, C.uint64_t(n), boolToInt(last)); s != C.CPB_OK {
			return nil, errors.New("csvplus: cpb_stream_push failed")
		}
		more, serr = collect()
		more = more && !last
		if serr != nil {
			break
		}
	}
	if len(parts) <= 1 {
		if len(parts) == 0 {
			return nil, serr
		}
		return parts[0], serr
	}
	hs := make([]*C.cpb_table, len(parts)+1)
	for i, p := range parts {
		hs[i] = p.h
	}
	var out *C.cpb_table
	if s := C.cpb_table_concat(c.h, &hs[0], C.int(len(parts)), &out); s != C.CPB_OK {
		return nil, errors.New("csvplus: cpb_table_concat failed")
	}
	runtime.KeepAlive(parts)
	return newTable(c, out), serr
}

func boolToInt(b bool) C.int {
	if b {
		return 1
	}
	return 0
}

// Iterate reads the input, converts every record to a Row and calls fn (csvplus.go:1080).  Rows delivered before a
// data error reach fn before the error is returned, like the streaming reference.
func (r *Reader) Iterate(fn RowFunc) error {
	return Take(r)(fn)
}
