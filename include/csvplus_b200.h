/* csvplus_b200.h — C ABI of the H100-native (sm_90a) csvplus hot path.
 *
 * The reference (maxim2266/csvplus, pure Go, single file csvplus.go) has no FFI seam;
 * its only boundary is the Go API (SURVEY.md §8b).  These entry points are exactly what a
 * cgo binding of that API needs for the data-parallel path
 *   Reader.Iterate -> SelectColumns -> Filter(Like/All/Any/Not) -> IndexOn/UniqueIndexOn -> Join -> ToCsv
 * Each entry point cites the reference code it replaces (csvplus.go:line).  The Go-side
 * stub that binds them is shown in INTEGRATION.md (and go/csvplus/, unbuilt: no Go toolchain).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes; no C++/torch types; no exceptions cross the boundary.
 *   - every call returns a cpb_status; data errors additionally fill a cpb_error whose
 *     (line, msg) reproduce the reference's DataSourceError{Line, Err} (csvplus.go:1230-1238).
 *   - a null ctx, handle or required out-parameter is answered with CPB_ERR_ARG (the reason in cpb_last_error when there
 *     is a ctx to keep it), never dereferenced; a cpb_error passed in is cleared first.  The *_free calls accept null.
 *   - handles (cpb_ctx / cpb_table / cpb_index) are owned by the library and released by the
 *     matching *_free.  Input byte buffers are borrowed for the duration of the call only.
 *   - every entry point selects the ctx's device (goroutines migrate between OS threads) and
 *     runs on the ctx's own CUDA stream; a ctx serialises its calls (one in flight).
 *   - there is NO CPU fallback: if the CUDA device or kernels are unavailable the call fails.
 */
#ifndef CSVPLUS_B200_H
#define CSVPLUS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CPB_ABI_VERSION 1
#define CPB_MAX_PARSE_COLS 16 /* columns extracted by one fused parse call (output + predicate columns) */
/* the largest cpb_pred tree the device compiles; a larger one fails with CPB_ERR_UNSUPPORTED */
#define CPB_PRED_MAX_TERMS 32 /* Like (column, literal) pairs whose column exists, and set terms */
#define CPB_PRED_MAX_OPS 64   /* postfix operations: one per Like pair and per set term, per AND / OR / NOT joining them,
                                 per empty All / Any */
#define CPB_PRED_MAX_DEPTH 48 /* All / Any / Not nodes above the deepest node (the Likes of a set term add none) */
/* Set terms (value lists: Any(Like{id: v1}, Like{id: v2}, ...)).  Inside an Any node, the direct Like children that compare
 * the same SET of column names (key order inside a Like does not matter; a Like naming one column twice never joins a
 * group) form a group.  A group of at least CPB_PRED_SET_MIN children is one set term: true for a row whose values of
 * those columns equal, byte for byte, the literals of some child of the group.  It counts as one term and one operation;
 * the node's other children compile as they would without the group, and everything is ORed.  A set term is evaluated as
 * an IndexOn over the table of the group's literal tuples, probed as Except probes an index.  So a group is a set term
 * only when that index can exist:
 *   - at most 16 columns, and
 *   - sum over the group's columns of (w + L(w)) <= 4096 bytes, w = the longest literal of the column in bytes,
 *     L(w) = 1 if w < 255, 2 if w < 65535, else 4 (the key image: every value padded to w, then its length).
 * A group that fails either compiles as separate Like terms.  When a column of a set term is absent from the row type the
 * term is a constant false (as each of its Likes would be).  Every tree within the limits above has at most 32 terms, so
 * no group in it reaches CPB_PRED_SET_MIN: such trees compile exactly as without set terms. */
#define CPB_PRED_SET_MIN 33

typedef struct cpb_ctx cpb_ctx;
typedef struct cpb_table cpb_table; /* columnar batch of rows: Arrow-style string columns in HBM */
typedef struct cpb_index cpb_index; /* csvplus Index (csvplus.go:610-614): table sorted on key columns */
typedef struct cpb_stream cpb_stream; /* an input parsed in batches of whole records */

typedef struct cpb_str {
    const char* ptr;
    uint64_t len;
} cpb_str;

typedef enum cpb_status {
    CPB_OK = 0,
    CPB_ERR_DATA = 1,        /* reference-visible data error; see cpb_error; partial result may be returned */
    CPB_ERR_ARG = 2,         /* argument misuse (the reference panics for most of these) */
    CPB_ERR_CUDA = 3,        /* CUDA runtime failure, message in cpb_error.msg */
    CPB_ERR_UNSUPPORTED = 4, /* option combination not yet lowered to kernels (documented in DESIGN.md) */
    CPB_ERR_NOMEM = 5
} cpb_status;

/* cpb_error.kind — one per reference error site */
typedef enum cpb_err_kind {
    CPB_E_NONE = 0,
    CPB_E_BARE_QUOTE = 1,       /* encoding/csv ErrBareQuote, via mapError csvplus.go:1209-1215 */
    CPB_E_QUOTE = 2,            /* encoding/csv ErrQuote */
    CPB_E_FIELD_COUNT = 3,      /* encoding/csv ErrFieldCount ("wrong number of fields") */
    CPB_E_INVALID_DELIM = 4,    /* "csv: invalid field or comment delimiter" */
    CPB_E_EOF = 5,              /* empty input while a header row is expected: "row 1: EOF" */
    CPB_E_EMPTY_HEADER = 6,     /* csvplus.go:1157 */
    CPB_E_MISPLACED_COLUMN = 7, /* csvplus.go:1179 */
    CPB_E_COLUMN_NOT_FOUND = 8, /* csvplus.go:1198/:1201 "column(s) not found: ..." */
    CPB_E_COLUMN_INDEX = 9,     /* csvplus.go:1128  column not found: %q (%d) */
    CPB_E_MISSING_COLUMN = 10,  /* csvplus.go:129/:145  missing column %q */
    CPB_E_MISSING_INDEX_COLUMN = 11, /* csvplus.go:725 */
    CPB_E_DUPLICATE_KEY = 12,   /* csvplus.go:751 */
    CPB_E_TOO_LARGE = 13,       /* a column/batch exceeds the 4 GiB-per-column batch limit (DESIGN.md) */
    CPB_E_CUDA = 14,
    CPB_E_UNSUPPORTED = 15,
    CPB_E_NUM_SYNTAX = 16,      /* csvplus.go:176/:198  cannot convert %q to integer|float: invalid syntax */
    CPB_E_NUM_RANGE = 17,       /* csvplus.go:176/:198  ...: value out of range */
    CPB_E_GOB = 18              /* LoadIndex (csvplus.go:683-705): the file is not an index gob stream ("EOF", "unexpected EOF", ...) */
} cpb_err_kind;

typedef struct cpb_error {
    int32_t kind;         /* cpb_err_kind */
    int32_t column_index; /* when a column is named: its position in the caller's list, else -1 */
    uint64_t line;        /* DataSourceError.Line: 1-based record ordinal incl. header (Reader, csvplus.go:1102-1137);
                             0-based row index for table sources (iterate, csvplus.go:243) */
    int32_t has_line;     /* 1 when the reference wraps the error as "row <line>: <msg>" */
    int32_t _pad;
    char msg[488];        /* the reference's inner error text, NUL-terminated */
} cpb_error;

/* Reader options — mirrors Reader{delimiter, comment, numFields, lazyQuotes, trimLeadingSpace,
 * headerFromFirstRow}, csvplus.go:924-931; defaults csvplus.go:962-968. */
typedef struct cpb_reader_opts {
    uint32_t delimiter;  /* rune; default ',' */
    uint32_t comment;    /* rune; 0 = none */
    int32_t num_fields;  /* 0 auto (first record), -1 any, n>0 exact (csvplus.go:1058-1076) */
    uint8_t lazy_quotes;
    uint8_t trim_leading_space;
    uint8_t header_from_first_row; /* 1: ExpectHeader/SelectColumns/none; 0: AssumeHeader */
    uint8_t _pad;
} cpb_reader_opts;

/* one entry of Reader.header map[string]int (csvplus.go:929): index -1 = find by name in record 1
 * (SelectColumns csvplus.go:1039-1056); >=0 = ExpectHeader / AssumeHeader position. */
typedef struct cpb_header_col {
    cpb_str name;
    int32_t index;
    int32_t _pad;
} cpb_header_col;

/* Predicate AST for the recognisable predicates Like/All/Any/Not (csvplus.go:1243-1293). */
enum { CPB_PRED_LIKE = 0, CPB_PRED_ALL = 1, CPB_PRED_ANY = 2, CPB_PRED_NOT = 3 };
typedef struct cpb_pred {
    int32_t op;
    int32_t n;                           /* LIKE: #pairs; ALL/ANY: #children; NOT: 1 */
    const cpb_str* keys;                 /* LIKE: column names */
    const cpb_str* values;               /* LIKE: literals */
    const struct cpb_pred* const* children;
} cpb_pred;

/* ------------------------------------------------------------------ context
 * A ctx = one device + one stream + one stream-ordered memory pool; calls on one ctx are serialised, several
 * ctxs (one per host thread) run concurrently.  Tables and indices belong to the ctx that created them and must
 * be freed before it is shut down.  An index may be probed (cpb_join / cpb_except) by tables of other ctxs of the
 * same device: what such a probe builds lazily inside the index is taken from the index owner's pool, so the
 * probing ctx may be shut down before the index; the RESULT table belongs to the probing ctx. */
int cpb_abi_version(void);
int cpb_init(int device, cpb_ctx** out);
void cpb_shutdown(cpb_ctx* ctx);
void* cpb_ctx_stream(cpb_ctx* ctx); /* the ctx's cudaStream_t (for event timing by the caller) */
int cpb_sync(cpb_ctx* ctx);
/* Maps `nbytes` of device memory into the ctx's pool ahead of time (one allocation + release; the pool keeps what it
 * maps).  Tables, indices and scratch of later calls are then carved out of memory the pool already holds: no call in a
 * steady loop waits for the driver to map pages.  Optional — the pool grows on demand without it (and then the first
 * iterations of a loop pay for the growth).  There is no counterpart in csvplus.go (Go's heap grows the same way). */
int cpb_pool_reserve(cpb_ctx* ctx, uint64_t nbytes);
const char* cpb_last_error(cpb_ctx* ctx); /* last CUDA / argument error text of this ctx */
/* *bytes = the most device memory the ctx's pool has had allocated at once since the last reset (reset != 0 then starts
 * a new window at the current use): the peak memory of a step, a stream, a test */
int cpb_pool_used_high(cpb_ctx* ctx, int reset, uint64_t* bytes);

/* Staging memory.  Host: pinned, the Go side fills it with io.ReadFull (replaces the 4 KB bufio reads
 * under csvplus.go:1091).  Device: zero-padded input buffer for callers that produce CSV bytes on the GPU. */
int cpb_host_alloc(cpb_ctx* ctx, uint64_t nbytes, void** out);
int cpb_host_free(cpb_ctx* ctx, void* p);
int cpb_device_alloc(cpb_ctx* ctx, uint64_t nbytes, void** out);
int cpb_device_free(cpb_ctx* ctx, void* p);
int cpb_memcpy_h2d(cpb_ctx* ctx, void* dst_dev, const void* src_host, uint64_t nbytes);
int cpb_memcpy_d2h(cpb_ctx* ctx, void* dst_host, const void* src_dev, uint64_t nbytes);

/* ------------------------------------------------------------------ parse (+select +filter)
 * Replaces Reader.Iterate (csvplus.go:1080-1146) + makeHeader (:1149-1206) + encoding/csv.Reader
 * (+ a directly following Filter of recognisable predicates, csvplus.go:276-286).
 *   bytes/nbytes : the whole CSV input; on_device=0: host memory (pinned or pageable), copied H2D inside;
 *                  on_device=1: device memory, 16-byte aligned, readable up to the next multiple of 16.
 *   spec/nspec   : Reader.header; nspec=0 => all columns named by record 1.
 *   filter       : nullable; rows failing it are never materialised.
 *   out          : table of the delivered rows (rows before the error when status==CPB_ERR_DATA).
 * Column order of the table = spec order (or file header order when nspec=0). */
int cpb_parse_csv(cpb_ctx* ctx, const void* bytes, uint64_t nbytes, int on_device, const cpb_reader_opts* opts,
                  const cpb_header_col* spec, int nspec, const cpb_pred* filter, cpb_table** out, cpb_error* err);

/* ------------------------------------------------------------------ streamed parse
 * Reader.Iterate over an input of any size (csvplus.go:1080-1146 pulls one record at a time): the input is pushed in
 * host pieces and parsed in batches of whole records, cut on the GPU at the end of the last complete record; the tail
 * is carried to the front of the next batch.  Concatenating the batches' tables gives cpb_parse_csv's rows, and the
 * first error and its line are cpb_parse_csv's (every line number and table first_line is global).
 *   open : reader options, header spec and fused filter as cpb_parse_csv; `filter` is borrowed until cpb_stream_free.
 *   push : appends bytes behind the carried tail; the host->device copy is enqueued on the stream's own copy stream and
 *          the call returns; host_bytes must stay untouched until the next cpb_stream_next returns.  is_last marks the
 *          end of the input (nbytes may be 0).
 *   next : parses the complete records pushed so far.  *out = NULL when there is none yet (push more); CPB_ERR_DATA with
 *          the rows before the error as in cpb_parse_csv; *done = 1 after the last batch or an error.  One host
 *          synchronisation for the cut, besides the parse's own.
 * The first batch must hold the whole first record (header): it grows until it does.  Device memory: two staging slots
 * of about one batch plus the longest record, and one batch's tables.  With CommentChar or LazyQuotes the cut takes the
 * record-boundary DFA of the general reader path. */
int cpb_stream_open(cpb_ctx* ctx, const cpb_reader_opts* opts, const cpb_header_col* spec, int nspec, const cpb_pred* filter,
                    cpb_stream** out, cpb_error* err);
int cpb_stream_push(cpb_stream* s, const void* host_bytes, uint64_t nbytes, int is_last);
int cpb_stream_next(cpb_stream* s, cpb_table** out, int* done, cpb_error* err);
void cpb_stream_free(cpb_stream* s);
/* the cut alone: the end of the last complete record of `bytes` (which start at a record start), 0 when there is none —
 * what cpb_stream_next parses of a buffer that is not the last (tests / timing) */
int cpb_csv_stream_cut(cpb_ctx* ctx, const void* bytes, uint64_t nbytes, int on_device, const cpb_reader_opts* opts, uint64_t* cut);

/* ------------------------------------------------------------------ tables */
int64_t cpb_table_num_rows(const cpb_table* t);
int cpb_table_num_cols(const cpb_table* t);
int cpb_table_col_name(const cpb_table* t, int col, cpb_str* out);
int cpb_table_find_col(const cpb_table* t, cpb_str name); /* -1 if absent (Row.HasColumn csvplus.go:62) */
int cpb_table_col_bytes(cpb_ctx* ctx, const cpb_table* t, int col, int64_t row_lo, int64_t row_hi, uint64_t* nbytes);
/* copy rows [row_lo,row_hi) of one column to host: offsets_out[row_hi-row_lo+1] (relative), data_out[cap] */
int cpb_table_fetch_column(cpb_ctx* ctx, const cpb_table* t, int col, int64_t row_lo, int64_t row_hi,
                           int64_t* offsets_out, uint8_t* data_out, uint64_t cap);
/* raw device views (valid while the table lives): offsets uint32[nrows+1], data bytes */
int cpb_table_column_device(const cpb_table* t, int col, const uint32_t** offsets, const uint8_t** data);
/* build a table from host columns (TakeRows, csvplus.go:218): offsets int64[nrows+1] per column */
int cpb_table_from_host(cpb_ctx* ctx, int ncols, const cpb_str* names, const int64_t* const* offsets,
                        const uint8_t* const* data, int64_t nrows, cpb_table** out);
/* build a table that adopts copies of device columns (multi-GPU all-gather import) */
int cpb_table_from_device(cpb_ctx* ctx, int ncols, const cpb_str* names, const uint32_t* const* offsets,
                          const uint8_t* const* data, int64_t nrows, cpb_table** out);
/* concatenate row-wise (same columns): used to assemble all-gathered shards */
int cpb_table_concat(cpb_ctx* ctx, const cpb_table* const* parts, int nparts, cpb_table** out);
/* DataSource.SelectColumns (csvplus.go:511-525) / DropColumns (:493-507): metadata only, buffers shared */
int cpb_table_select(cpb_ctx* ctx, const cpb_table* t, const cpb_str* cols, int n, cpb_table** out, cpb_error* err);
int cpb_table_drop(cpb_ctx* ctx, const cpb_table* t, const cpb_str* cols, int n, cpb_table** out);
/* DataSource.Filter with Like/All/Any/Not (csvplus.go:276-286, :1243-1293) */
int cpb_table_filter(cpb_ctx* ctx, const cpb_table* t, const cpb_pred* pred, cpb_table** out);
/* DataSource.TakeWhile / DropWhile (csvplus.go:346-374) with a recognisable predicate: the first row for which it is
 * false (the row count when there is none); TakeWhile = cpb_table_slice(0, row), DropWhile = cpb_table_slice(row, n) */
int cpb_table_first_false(cpb_ctx* ctx, const cpb_table* t, const cpb_pred* pred, int64_t* row);
/* Top(n)/Drop(n) as row-range views (csvplus.go:313-342) */
int cpb_table_slice(cpb_ctx* ctx, const cpb_table* t, int64_t row_lo, int64_t row_hi, cpb_table** out);
void cpb_table_free(cpb_table* t);

/* ------------------------------------------------------------------ index
 * IndexOn / UniqueIndexOn = createIndex / createUniqueIndex (csvplus.go:527-537, :707-756):
 * validates key columns, sorts by bytewise per-column order (indexImpl.Less :794-807); ties keep
 * input order (the reference's sort.Sort is unstable: SURVEY §Q2).  unique!=0 adds the adjacent
 * duplicate check and fails with CPB_E_DUPLICATE_KEY naming the lowest duplicated key. */
int cpb_index_build(cpb_ctx* ctx, const cpb_table* t, const cpb_str* key_cols, int nkeys, int unique,
                    cpb_index** out, cpb_error* err);
int64_t cpb_index_num_rows(const cpb_index* ix);
int cpb_index_num_keys(const cpb_index* ix);
/* the sorted rows as a table (Index.Iterate csvplus.go:618-620); borrowed view, free with cpb_table_free */
int cpb_index_table(cpb_ctx* ctx, const cpb_index* ix, cpb_table** out);
/* Index.Find (csvplus.go:625-627, :870-891): rows whose leading key columns equal values */
int cpb_index_find(cpb_ctx* ctx, const cpb_index* ix, const cpb_str* values, int n, cpb_table** out);
/* Index.SubIndex (csvplus.go:632-641) */
int cpb_index_sub(cpb_ctx* ctx, const cpb_index* ix, const cpb_str* values, int n, cpb_index** out);
/* Index.ResolveDuplicates (csvplus.go:651-653, dedup :810-867), split around the opaque Go callback:
 * groups(): offsets of every run of >=2 equal keys in sorted order: group g = rows [lo[g], hi[g]).
 * apply(): keep[g] = absolute sorted row to keep for group g, or -1 to drop the group ("empty row").
 * The reference's trailing-singleton loss (SURVEY §Q1) is reproduced when bug_compatible!=0. */
int cpb_index_dup_groups(cpb_ctx* ctx, const cpb_index* ix, int64_t* ngroups, int64_t** lo, int64_t** hi);
int cpb_index_dedup_apply(cpb_ctx* ctx, cpb_index* ix, int64_t ngroups, const int64_t* keep, int bug_compatible);
/* same, and keep[g] <= -2 puts row (-2 - keep[g]) of `replacements` in the place of group g: the resolver may return a
 * row that is not one of the group's rows (csvplus.go:838-848 stores whatever row came back, without re-sorting).
 * `replacements` must have the columns of the index rows; nullable when no keep[g] <= -2. */
int cpb_index_dedup_apply2(cpb_ctx* ctx, cpb_index* ix, int64_t ngroups, const int64_t* keep, const cpb_table* replacements,
                           int bug_compatible, cpb_error* err);
void cpb_free(void* p); /* releases arrays returned by cpb_index_dup_groups / cpb_table_to_csv */
void cpb_index_free(cpb_index* ix);
/* key column k of the index (index.impl.columns[k]); valid while the index lives */
int cpb_index_key_col(const cpb_index* ix, int k, cpb_str* out);

/* ------------------------------------------------------------------ index files (encoding/gob)
 * Index.WriteTo (csvplus.go:655-680): the gob stream of `columns []string` then `rows []Row`, the rows in the index's
 * stored order, the pairs of a row in bytewise column-name order.  The file = the prefix, then the rows in row-range
 * batches.
 *   begin : *prefix_len = the bytes before the first row (type definitions, the columns value, the rows message header),
 *           written to prefix when they fit cap (else CPB_ERR_ARG, nothing written); *total_len = the whole file.  A rows
 *           message that encoding/gob's decoder would refuse (8 GiB or more) fails here: CPB_ERR_DATA / CPB_E_TOO_LARGE.
 *   into  : rows [row_lo, row_hi) into caller-owned (pinned) host memory; cap too small: CPB_ERR_ARG with *nbytes = the
 *           size needed, nothing written.  One call produces less than 4 GiB (else CPB_ERR_DATA / CPB_E_TOO_LARGE).
 * LoadIndex (csvplus.go:683-705): an index from the bytes of a whole file.  Type ids and definition order are free, and
 * so is the pair order of every row; the rows are decoded on the GPU.  The index holds the rows in file order (Find /
 * Join / Except search them as the reference does, sorted or not) and is not marked unique.  A stream that is not an
 * index file fails with CPB_ERR_DATA / CPB_E_GOB: msg "EOF" (no message where one is due), "unexpected EOF" (a cut
 * message) or a description; so do rows whose column sets differ.  Limits: at most 256 columns per row, each column
 * of the loaded rows below 4 GiB (CPB_E_TOO_LARGE). */
int cpb_index_gob_begin(cpb_ctx* ctx, const cpb_index* ix, void* prefix, uint64_t cap, uint64_t* prefix_len, uint64_t* total_len,
                        cpb_error* err);
int cpb_index_gob_into(cpb_ctx* ctx, const cpb_index* ix, int64_t row_lo, int64_t row_hi, void* host_dst, uint64_t cap,
                       uint64_t* nbytes, cpb_error* err);
int cpb_index_load_gob(cpb_ctx* ctx, const void* bytes, uint64_t nbytes, cpb_index** out, cpb_error* err);

/* ------------------------------------------------------------------ join
 * DataSource.Join (csvplus.go:545-583): inner join of probe rows against the index on probe_cols
 * (n=0: natural join on the index key names); n < #keys is a prefix match.  Output rows in probe
 * order, then index order; columns = index columns U probe columns, probe wins name collisions
 * (mergeRows :571-583).  A probe table lacking a join column fails with CPB_E_MISSING_COLUMN at row 0. */
int cpb_join(cpb_ctx* ctx, const cpb_table* probe, const cpb_index* ix, const cpb_str* probe_cols, int n,
             cpb_table** out, cpb_error* err);
/* DataSource.Except (csvplus.go:588-608): probe rows whose key is absent from the index */
int cpb_except(cpb_ctx* ctx, const cpb_table* probe, const cpb_index* ix, const cpb_str* probe_cols, int n,
               cpb_table** out, cpb_error* err);

/* ------------------------------------------------------------------ ToCsv
 * DataSource.ToCsv (csvplus.go:379-406) + encoding/csv.Writer defaults: header line, then one line
 * per row with the named columns; bytes returned in a pinned host buffer (release with cpb_host_free). */
int cpb_table_to_csv(cpb_ctx* ctx, const cpb_table* t, const cpb_str* cols, int n, void** bytes, uint64_t* nbytes,
                     cpb_error* err);
/* same, result left in device memory (release with cpb_device_free) */
int cpb_table_to_csv_device(cpb_ctx* ctx, const cpb_table* t, const cpb_str* cols, int n, void** dev_bytes,
                            uint64_t* nbytes, cpb_error* err);

/* one batch of a streamed ToCsv/ToCsvFile (csvplus.go:379-443) into caller-owned (pinned) host memory: the header
 * line is written only when with_header != 0 (the csv.Writer writes it once, before the first batch, :387);
 * nothing is allocated per call, the device->host copy runs on the ctx stream and the call returns when it is done. */
int cpb_table_to_csv_into(cpb_ctx* ctx, const cpb_table* t, const cpb_str* cols, int n, int with_header, void* host_dst,
                          uint64_t cap, uint64_t* nbytes, cpb_error* err);

/* ------------------------------------------------------------------ ToJSON
 * DataSource.ToJSON (csvplus.go:446-474) of one table or one batch of a streamed result: every column, keys sorted
 * bytewise, encoding/json's string escaping with SetEscapeHTML(false), one object per line.
 * first_batch: the first row is preceded by '[' (else ','); last_batch: ']' is appended.  first=last=1 on an empty
 * table gives "[]".  One call produces less than 4 GiB (else CPB_ERR_DATA / CPB_E_TOO_LARGE: write row-range batches). */
int cpb_table_to_json(cpb_ctx* ctx, const cpb_table* t, int first_batch, int last_batch, void** bytes, uint64_t* nbytes,
                      cpb_error* err); /* pinned host bytes: release with cpb_host_free */
int cpb_table_to_json_device(cpb_ctx* ctx, const cpb_table* t, int first_batch, int last_batch, void** dev_bytes,
                             uint64_t* nbytes, cpb_error* err); /* device bytes: release with cpb_device_free */
/* into caller-owned (pinned) host memory; cap too small: CPB_ERR_ARG with *nbytes = the size needed, nothing written */
int cpb_table_to_json_into(cpb_ctx* ctx, const cpb_table* t, int first_batch, int last_batch, void* host_dst, uint64_t cap,
                           uint64_t* nbytes, cpb_error* err);

/* ------------------------------------------------------------------ numeric columns
 * Row.ValueAsInt / Row.ValueAsFloat64 (csvplus.go:163-205: strconv.Atoi / strconv.ParseFloat(s, 64), Go 1.23) of every
 * row of one column, into caller-owned device memory, stream-ordered on the ctx stream; returns after one host
 * synchronisation.  values[nrows] is always written (Go's value on error too: 0 for a syntax error, the clamped integer
 * or +-Inf for a range error); status[nrows] is nullable (CPB_NUM_*); *nbad = failing rows.
 * nbad > 0: CPB_ERR_DATA, kind CPB_E_NUM_SYNTAX / CPB_E_NUM_RANGE of the first failing row, err->line = that row
 * (0-based), has_line = 0, msg = the reference's text.  An absent column on a non-empty table: CPB_ERR_DATA,
 * CPB_E_MISSING_COLUMN, line 0, has_line = 0.  A float column converts at most 2^32 - 1 rows per call. */
enum { CPB_NUM_OK = 0, CPB_NUM_SYNTAX = 1, CPB_NUM_RANGE = 2 };
int cpb_table_column_as_int64(cpb_ctx* ctx, const cpb_table* t, cpb_str column, int64_t* values, uint8_t* status,
                              uint64_t* nbad, cpb_error* err);
int cpb_table_column_as_float64(cpb_ctx* ctx, const cpb_table* t, cpb_str column, double* values, uint8_t* status,
                                uint64_t* nbad, cpb_error* err);

/* ------------------------------------------------------------------ computed columns
 * The reference's Map(func(row) Row { row[column] = value; return row }) over every row: *out = t with `column` set,
 * replaced in place when t has it, else appended.  Every other column shares t's buffers (row-range views too); t is
 * not modified.  dev_values[nrows] is device memory, read on the ctx stream (the caller orders its producer before
 * the call); it may be released once the call returns.
 *   set_int64  : strconv.FormatInt(v, 10).
 *   set_float64: strconv.FormatFloat(x, fmt, prec, 64), byte for byte; fmt one of e E f g G, prec -1..64 (-1: the
 *                shortest digits that read back as x).  Another fmt or prec: CPB_ERR_ARG, nothing computed.
 *   set_literal: value in every row.
 * One column stays below 4 GiB: a column of 4 GiB or more fails with CPB_ERR_DATA / CPB_E_TOO_LARGE (checked on the
 * exact 64-bit total, before any offset is written).  Host synchronisations: none for an empty table; for set_float64
 * one, or two when some row needs the exact big-integer path (its kernel, format_rare, then shows in cpb_stats_get).
 * filter_flags: the rows whose dev_keep[row] byte is nonzero, in order (dev_keep[nrows] read on the ctx stream). */
int cpb_table_set_int64(cpb_ctx* ctx, const cpb_table* t, cpb_str column, const int64_t* dev_values, cpb_table** out, cpb_error* err);
int cpb_table_set_float64(cpb_ctx* ctx, const cpb_table* t, cpb_str column, const double* dev_values, char fmt, int prec,
                          cpb_table** out, cpb_error* err);
int cpb_table_set_literal(cpb_ctx* ctx, const cpb_table* t, cpb_str column, cpb_str value, cpb_table** out, cpb_error* err);
int cpb_table_filter_flags(cpb_ctx* ctx, const cpb_table* t, const uint8_t* dev_keep, cpb_table** out, cpb_error* err);

/* ------------------------------------------------------------------ multi-GPU (SURVEY §8e)
 * The probe stream shards by row range with no data-path collective; the one exchange step is the all-gather of the
 * build-side columns (each rank parses 1/N of the build file) so that every rank can build the full Index
 * (csvplus.go:707-767) — the reference has no counterpart, it is single-threaded (csvplus.go:33-46).  Transport: NCCL
 * over NVLink, bound at run time (libnccl.so.2).
 *   one process per GPU : rank 0 calls cpb_comm_unique_id, the host distributes the 128 bytes (any side channel), every
 *                         rank calls cpb_comm_init_rank on its own ctx; cpb_allgather_table is then a collective.
 *   one process, n GPUs : cpb_init_multi creates n ctxs sharing one communicator (a Go program would use this form);
 *                         cpb_allgather_tables drives all ranks from one thread, or cpb_allgather_table is called
 *                         from one host thread per ctx.
 * cpb_allgather_table returns on every rank the concatenation of all ranks' rows in rank order (= input order of
 * row-range shards).  Row-range views are accepted.  One host synchronisation (the sizes).
 * cpb_allgather_u64 exchanges `count` host values per rank (byte-range shards of one file exchange their quote parity
 * and record counts with it, see cpb_parse_csv_shard); without a communicator it copies in to out. */
#define CPB_UNIQUE_ID_BYTES 128
int cpb_comm_unique_id(uint8_t* id128);
int cpb_comm_init_rank(cpb_ctx* ctx, int nranks, int rank, const uint8_t* id128);
int cpb_init_multi(const int* devices, int n, cpb_ctx** out /* [n] */);
int cpb_comm_size(cpb_ctx* ctx);
int cpb_comm_rank(cpb_ctx* ctx);
int cpb_allgather_table(cpb_ctx* ctx, const cpb_table* local, cpb_table** out);
int cpb_allgather_tables(cpb_ctx* const* ctxs, const cpb_table* const* locals, int n, cpb_table** outs /* [n] */);
int cpb_allgather_u64(cpb_ctx* ctx, const uint64_t* in, int count, uint64_t* out /* [nranks * count] */);
/* layout arithmetic of the all-gather-v alone (pure host code): meta[q] = {rows, (first, end) byte offset per column}
 * of rank q -> row_base[nranks+1], byte_base[ncols][nranks+1] */
int cpb_allgather_layout(int nranks, int ncols, const uint64_t* meta, uint64_t* row_base, uint64_t* byte_base);

/* Byte-range shards of ONE file (SURVEY §8e): rank r holds the bytes [lo_r, hi_r + look-ahead) of the file, lo_0 = 0,
 * lo_{r+1} = hi_r.  A record belongs to the shard in whose (lo, hi] its first byte lies (shard 0 also owns byte 0), so no
 * look-behind is needed; the look-ahead must reach the end of the record that starts at hi (else CPB_ERR_ARG).
 *   1. every rank: cpb_csv_quote_parity over its own [lo, hi)          -> q_r
 *   2. all-gather of q (cpb_allgather_u64); initial_parity_r = XOR of q_s, s < r
 *   3. every rank: cpb_parse_csv_shard(..., own_bytes = hi - lo, shard_index = r, is_last, initial_parity_r, ...)
 *      -> its rows (concatenation in rank order = the reference's row order) and `records` (owned records, pre-filter)
 *   4. all-gather of (records, failed, local line): DataSourceError.Line = base (2 with a header row, else 1) + records of
 *      the shards before the first failing one + its local line (csvplus.go:1102-1137); later shards drop their rows.
 * Shards after the first need the resolved header: header_from_first_row = 0, spec = (name, index) pairs, and an explicit
 * num_fields (the count of the file's first record, or -1).  Default reader options only.  On CPB_ERR_DATA err->line is
 * the LOCAL 0-based ordinal of the failing record among this shard's records. */
/* of a table that cpb_parse_csv produced: the field index column `col` was read from, and the number of fields of the
 * file's first record (-1 when the table did not come from the parser) — the resolved header for shards after the first */
int cpb_table_col_field(const cpb_table* t, int col);
int cpb_table_record_fields(const cpb_table* t);
int cpb_csv_quote_parity(cpb_ctx* ctx, const void* bytes, uint64_t nbytes, int on_device, uint32_t* parity);
int cpb_parse_csv_shard(cpb_ctx* ctx, const void* bytes, uint64_t nbytes, int on_device, uint64_t own_bytes, int shard_index, int is_last,
                        uint32_t initial_parity, const cpb_reader_opts* opts, const cpb_header_col* spec, int nspec,
                        const cpb_pred* filter, cpb_table** out, uint64_t* records, cpb_error* err);

/* ------------------------------------------------------------------ measurement
 * Per-kernel launch records of this ctx since the last reset: name, launches, device ms (CUDA events on
 * the ctx stream) and algorithmic bytes, for the roofline JSON of bench.py. */
typedef struct cpb_kstat {
    char name[48];
    uint64_t launches;
    double ms;
    uint64_t algo_bytes;
} cpb_kstat;
int cpb_stats_enable(cpb_ctx* ctx, int on);
int cpb_stats_reset(cpb_ctx* ctx);
int cpb_stats_get(cpb_ctx* ctx, cpb_kstat* out, int cap, int* n);
uint64_t cpb_kernel_launches(cpb_ctx* ctx); /* total kernels this ctx has launched */
uint64_t cpb_host_syncs(cpb_ctx* ctx);      /* blocking host waits on the ctx stream issued by the library so far */

/* ------------------------------------------------------------------ synthetic data (bench / tests only)
 * Deterministic generators of SURVEY §8(d) tables, written on the GPU into a device buffer obtained from
 * cpb_device_alloc.  kind: 0 people/customers, 1 orders, 2 products.  Rows [row_lo,row_hi); header line
 * iff with_header.  permute!=0 writes ids through a seeded bijection.  Call with dst=NULL to size. */
int cpb_gen_csv(cpb_ctx* ctx, int kind, uint64_t seed, uint64_t row_lo, uint64_t row_hi, uint64_t n_cust,
                uint64_t n_prod, int with_header, int permute, void* dst, uint64_t cap, uint64_t* nbytes);

#ifdef __cplusplus
}
#endif
#endif /* CSVPLUS_B200_H */
