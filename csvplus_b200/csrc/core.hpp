// core.hpp — host-side internals shared by the C-ABI translation units:
// context (device, stream, stream-ordered pool), refcounted device buffers, string columns,
// tables, indices, error helpers and per-kernel timing records.
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <optional>
#include <string>
#include <vector>

#include "../../include/csvplus_b200.h"

namespace cpb {

struct Ctx;

// ------------------------------------------------------------------ errors
struct CudaFail { cudaError_t e; const char* what; const char* file; int line; };
#define CPB_CUDA(x)                                                        \
    do {                                                                   \
        cudaError_t _e = (x);                                              \
        if (_e != cudaSuccess) throw ::cpb::CudaFail{_e, #x, __FILE__, __LINE__}; \
    } while (0)

struct DataError {  // reference-visible error (cpb_error payload)
    int kind; int column_index; uint64_t line; bool has_line; std::string msg;
};
struct ArgError { int status; std::string msg; };

inline void fill_error(cpb_error* e, int kind, int col, uint64_t line, bool has_line, const std::string& msg) {
    if (!e) return;
    e->kind = kind; e->column_index = col; e->line = line; e->has_line = has_line ? 1 : 0; e->_pad = 0;
    size_t n = msg.size() < sizeof(e->msg) - 1 ? msg.size() : sizeof(e->msg) - 1;
    memcpy(e->msg, msg.data(), n); e->msg[n] = 0;
}
inline void clear_error(cpb_error* e) { if (e) { memset(e, 0, sizeof(*e)); e->column_index = -1; } }

// Go's %q for the plain names csvplus prints (csvplus.go:129, :725, :1128, :1179)
std::string go_quote(const std::string& s);

// ------------------------------------------------------------------ device memory
struct DevBuf {  // stream-ordered allocation owned by a ctx
    Ctx* ctx = nullptr; void* p = nullptr; size_t n = 0;
    DevBuf(Ctx* c, size_t bytes);
    // memory of `owner`'s pool, allocated in the stream order of `user` (usable by user's kernels at once) and
    // released on owner's stream: for structures another context builds lazily inside an object owner owns
    DevBuf(Ctx* owner, Ctx* user, size_t bytes);
    struct Borrow {};
    DevBuf(Borrow, const void* ptr, size_t bytes) : ctx(nullptr), p(const_cast<void*>(ptr)), n(bytes) {}  // caller-owned memory: never freed here
    ~DevBuf();
    DevBuf(const DevBuf&) = delete; DevBuf& operator=(const DevBuf&) = delete;
    template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};
using Buf = std::shared_ptr<DevBuf>;

// Arrow-style string column: value i = data[offsets[i] .. offsets[i+1]); offsets are uint32 (a
// column of one table/batch holds < 4 GiB of bytes — DESIGN.md "batches").  `row0` lets row-range
// views (Top/Drop/Find/SubIndex) share the buffers.
struct Column {
    std::string name;
    Buf offsets;      // uint32[nrows_alloc+1]
    Buf data;         // uint8[]
    int64_t row0 = 0; // first row of this view inside `offsets`
    const uint32_t* off() const { return offsets->as<uint32_t>() + row0; }
    const uint8_t* bytes() const { return data ? data->as<uint8_t>() : nullptr; }
};

struct Table {
    Ctx* ctx = nullptr;
    int64_t nrows = 0;
    uint64_t first_line = 0;  // DataSourceError.Line the source reports for row 0 (csvplus.go:1137 / :243)
    std::vector<Column> cols;
    // set by the parser: the field index every column was read from and the field count of the file's first record —
    // what the shards of a file after the first need instead of the header row (cpb_parse_csv_shard)
    std::vector<int> src_field;
    int record_fields = 0;
    int find(const std::string& name) const {
        for (size_t i = 0; i < cols.size(); i++) if (cols[i].name == name) return (int)i;
        return -1;
    }
};

// "Built on some context's stream": what several contexts may use (the lazily built structures of an index) carries the
// event recorded after its last kernel; a user makes its own stream wait for it — no host synchronisation.
struct ReadyEvent {
    cudaEvent_t ev = nullptr;
    ~ReadyEvent() { if (ev) cudaEventDestroy(ev); }
};
using Ready = std::shared_ptr<ReadyEvent>;

// The order of the index rows that probe tables and row slots refer to: sorted (ix.image, ix.perm / ix.table) or as
// given (ix.derived.uimage, ix.src: a lazily sorted unique index)
enum class RowOrder { sorted, source };

// Probe table over the runs of equal prefixes of the first nk key columns (join.cu); run j = rows [heads[j], heads[j+1]).
// smem / global: uint32 slots holding j (0xFFFFFFFF = empty, linear probing), the key compared with the key image at
// heads[j]; smem when slots + heads fit 200 KB of shared memory.  unique16: 16-byte slots {12 key bytes, row + 1}, every
// run one row.  run32: 32-byte slots {24 key bytes, first row | run length << 32}.
struct ProbeTable {
    enum class Kind { smem, global, unique16, run32 };
    Kind kind = Kind::smem;
    Ready ready;
    uint32_t pbytes = 0;     // image bytes of the prefix
    uint64_t nslots = 0;     // slots of `kind`
    Buf slots;
    uint64_t nheads = 0;     // runs
    Buf heads;               // uint32[nheads+1]; heads[nheads] = nrows
};
// Row slots (gather.cu): the output columns of the index rows re-laid as one fixed-size slot per row (their
// bytes back to back) + one packed word of lengths per row, so that a join fetches an index row with ONE random
// access instead of two per column.  Built lazily per set of output columns when every value is short.
struct RowSlots {
    Ready ready;
    bool usable = false;
    uint32_t S = 0;   // slot bytes (multiple of 16, <= 64)
    Buf slots;        // uint8[nrows][S]
    Buf lens;         // uint32[nrows]: length of column c in bits 8c..8c+7
};
// Row-carrying hash table of a unique index whose full-key image is <= 12 bytes and whose other columns (at most 4) take
// <= 16 bytes in every row: one 32-byte slot (one DRAM sector) per entry holds the key, the lengths of those columns
// and their bytes (RowSlot, rowhash.cuh), so a full-key Join finds key, lengths and payload with ONE random access.
// Built by UniqueIndexOn (the build is the duplicate check) and complete when the index is returned: read-only after.
// Layout: nslots / region regions of `region` consecutive slots.  A key's probe sequence starts at slot_of(hash, nslots)
// and wraps from the last slot of that slot's region to the region's first, never into the next region; so each region
// is built on its own in shared memory, and a region can hold at most region - 1 keys.
struct RowHash {
    uint64_t nslots = 0;    // a multiple of region, at least 2 * rows + 16 (load factor about 1/2)
    uint32_t region = 0;    // slots per region: a power of two, RH_REGION (rowhash.cuh) unless the table is smaller
    Buf slots;              // RowSlot[nslots]; null = the index has no row-carrying table
    std::vector<int> cols;  // payload: every non-key column of the source, in schema order
};
// csvplus Index (csvplus.go:610-614, :785-788): rows sorted on `key_cols`.
struct Index {
    Ctx* ctx = nullptr;
    // The sorted rows exist in two forms.  A join needs neither the sorted columns nor their offsets: it probes the
    // hash table (built from the sorted key image) and fetches payload through row slots laid out straight from the
    // source rows + the sort permutation.  So the index build keeps (src, perm) and the physically sorted table is
    // materialised only when something iterates / looks up / dedups the index (sorted_table()).
    std::shared_ptr<Table> src;        // the rows as they were given to IndexOn (unsorted); null after a dedup
    Buf perm;                          // uint32[nrows]: sorted position -> row of src
    int64_t nrows = 0;
    std::shared_ptr<Table> table;      // sorted rows (lazily materialised, under `mu`)
    // A UNIQUE index whose duplicate check passed is not even sorted until something needs the order (iteration, Find,
    // SubIndex, a prefix join, dedup): a full-key join only needs "key -> row".  `sorted` tells whether perm / image
    // exist yet (ensure_sorted()).
    bool sorted = true;
    const Table& schema() const { return table ? *table : *src; }  // column names / count only
    bool unique = false;               // built by UniqueIndexOn and verified: every full key occurs once
    // false when the stored rows are not in key order (ResolveDuplicates with replacement rows, LoadIndex of such a file):
    // Join / Except then search the rows exactly as the reference's binary search does instead of probing a hash table
    bool in_order = true;
    std::vector<std::string> key_cols; // index.impl.columns
    std::vector<int> key_col_idx;      // positions in table->cols
    std::vector<uint32_t> key_width;   // per key column: max value length (bytes) in this index
    uint32_t image_words = 0;          // uint64 words per row of the key image
    Buf image;                         // uint64[image_words][nrows] (word-major / SoA): key image of the sorted rows
    // Built from the stored rows and dropped together by whatever replaces them (reset_derived()).  uimage: the key
    // image in source order of a unique index without a row-carrying table; the full-key probe table over it is the
    // duplicate check (every key must find itself) and serves full-key joins (join_order(), join.cu).
    struct Derived {
        Buf uimage;
        RowHash rowhash;
        std::map<std::pair<RowOrder, int>, ProbeTable> probe;                // by (order, leading key columns)
        std::map<std::pair<RowOrder, std::vector<int>>, RowSlots> row_slots;  // by (order, output columns)
    } derived;                         // (the maps are filled lazily, under `mu`)
    void reset_derived() { derived = Derived{}; }
    std::mutex mu;                     // several contexts may probe one index concurrently
};

// ------------------------------------------------------------------ kernel stats
struct KStat { uint64_t launches = 0; double ms = 0; uint64_t bytes = 0; };
struct PendingEvent { std::string name; cudaEvent_t a, b; uint64_t bytes; };

struct Ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaMemPool_t pool = nullptr;
    bool own_pool = false;
    std::mutex mu;              // one call in flight per ctx
    std::string last_error;
    int sm_count = 132;
    size_t smem_optin = 0;
    // stats
    bool stats_on = false;
    std::map<std::string, KStat> stats;
    std::vector<PendingEvent> pending;
    std::vector<cudaEvent_t> event_pool;  // recycled timing events
    uint64_t launches = 0;
    // small pinned scratch for D2H of results
    void* pinned = nullptr; size_t pinned_n = 0;
    // multi-GPU (comm.cu): ncclComm_t of this rank, null for a single-GPU ctx
    void* comm = nullptr; int nranks = 1, rank = 0; bool comm_owned = false;
    Ctx* alloc_for = nullptr;  // see dev_alloc
    // host synchronisations this ctx has issued (cudaStreamSynchronize on its stream): a pipeline step should need few
    uint64_t host_syncs = 0;

    void* pinned_scratch(size_t n);
    void drain_events();
    void harvest_events();
};

// RAII: time a kernel (or a group of launches) on the ctx stream when stats are enabled
struct KernelTimer {
    Ctx* c; bool on; cudaEvent_t a{}, b{}; std::string name; uint64_t bytes; int nlaunch;
    KernelTimer(Ctx* ctx, const char* nm, uint64_t algo_bytes, int launches = 1);
    ~KernelTimer();
};

// every blocking wait of the host on a ctx stream goes through here and is counted (cpb_host_syncs): a pipeline step
// should need few of them
inline void sync_stream(Ctx* c) {
    c->host_syncs++;
    CPB_CUDA(cudaStreamSynchronize(c->stream));
}

// device-to-host readback of one value / n values through the pinned scratch, with one (counted) synchronisation; the
// values are returned, so nothing keeps pointing into the scratch the next readback reuses
template <class T> T read_back(Ctx* c, const void* dev) {
    T* h = static_cast<T*>(c->pinned_scratch(sizeof(T)));
    CPB_CUDA(cudaMemcpyAsync(h, dev, sizeof(T), cudaMemcpyDeviceToHost, c->stream));
    sync_stream(c);
    return *h;
}
template <class T> std::vector<T> read_back(Ctx* c, const void* dev, size_t n) {
    T* h = static_cast<T*>(c->pinned_scratch(n * sizeof(T)));
    if (n) CPB_CUDA(cudaMemcpyAsync(h, dev, n * sizeof(T), cudaMemcpyDeviceToHost, c->stream));
    sync_stream(c);
    return std::vector<T>(h, h + n);
}

inline uint32_t nblk(uint64_t n, int threads) { return (uint32_t)((n + threads - 1) / threads); }  // grid size

inline Ready record_ready(Ctx* c) {
    auto r = std::make_shared<ReadyEvent>();
    CPB_CUDA(cudaEventCreateWithFlags(&r->ev, cudaEventDisableTiming));
    CPB_CUDA(cudaEventRecord(r->ev, c->stream));
    return r;
}
inline void wait_ready(Ctx* c, const Ready& r) { if (r && r->ev) CPB_CUDA(cudaStreamWaitEvent(c->stream, r->ev, 0)); }

struct DeviceGuard {  // every entry point: select device, serialise on the ctx
    std::unique_lock<std::mutex> lk;
    explicit DeviceGuard(Ctx* c) : lk(c->mu) { cudaSetDevice(c->device); }
};

inline Buf dev_alloc_owned(Ctx* owner, Ctx* user, size_t bytes) { return std::make_shared<DevBuf>(owner, user, bytes ? bytes : 1); }
// (while a ctx builds something that stays inside an object another ctx owns, its allocations come from that owner's pool)
inline Buf dev_alloc(Ctx* c, size_t bytes) {
    if (c->alloc_for && c->alloc_for != c) return dev_alloc_owned(c->alloc_for, c, bytes);
    return std::make_shared<DevBuf>(c, bytes ? bytes : 1);
}

inline std::string to_string(cpb_str s) { return std::string(s.ptr ? s.ptr : "", (size_t)s.len); }

// a table over rows [lo, hi) of t that shares t's buffers: every column, or the columns `pick` in that order.
// first_line stays at its default; the caller sets it where the rows keep the lines of their source
inline std::shared_ptr<Table> table_view(Ctx* c, const Table& t, int64_t lo, int64_t hi, const std::vector<int>* pick = nullptr) {
    auto r = std::make_shared<Table>(); r->ctx = c; r->nrows = hi - lo;
    for (size_t i = 0; i < (pick ? pick->size() : t.cols.size()); i++) {
        Column col = t.cols[pick ? (size_t)(*pick)[i] : i];
        col.row0 += lo;
        r->cols.push_back(col);
    }
    return r;
}

// ------------------------------------------------------------------ the extern "C" boundary
// A bad argument of an entry point (a null handle, a null out-parameter): CPB_ERR_ARG, `what` in cpb_last_error
inline void need(bool ok, const char* what) { if (!ok) throw ArgError{CPB_ERR_ARG, what}; }
// exception -> status translation used by every extern "C" body; c may be null (no context to record the text in)
int translate_exception(Ctx* c, cpb_error* err);
template <class F> int translated(Ctx* c, cpb_error* err, F&& body) {
    try { return body(); } catch (...) { return translate_exception(c, err); }
}
// Every entry point that works on a context runs as guarded(ctx, err, body): *err is cleared first, a null context is
// CPB_ERR_ARG, the context's device is selected and its calls serialised, and body(Ctx*) returns the status or throws
template <class F> int guarded(Ctx* c, cpb_error* err, F&& body) {
    clear_error(err);
    if (!c) return CPB_ERR_ARG;
    DeviceGuard g(c);
    return translated(c, err, [&]() -> int { return body(c); });
}

// ------------------------------------------------------------------ cross-TU operations
// parse.cu
struct ShardArgs {  // byte-range shard of one file (cpb_parse_csv_shard)
    uint64_t own_bytes;  // records starting at buffer positions (0, own_bytes] are this shard's ([0, own_bytes] for index 0)
    int index;           // 0 = the shard holding the start of the file
    bool is_last;        // the buffer ends where the file ends
    uint32_t pin0;       // parity of the quote bytes of the file before this buffer
};
// One parse: the rows before the first data error (all of them when there is none) and that error, as the reference
// delivers them; the record counts are what a shard or a batch of a stream adds to the records before it.
struct Parsed {
    std::shared_ptr<Table> table;
    std::optional<DataError> error;
    uint64_t records = 0;    // data records of the input (before filtering)
    bool no_record = false;  // the input holds no record at all (only blank or comment lines)
};
// line_base: DataSourceError.Line of the input's first data record (2 after a header row, 1 without; a later batch of a
// stream continues the count)
Parsed parse_csv(Ctx* c, const uint8_t* dev_bytes, uint64_t n, const cpb_reader_opts& o, const std::vector<std::pair<std::string, int>>& spec,
                 const cpb_pred* filter, uint64_t line_base, const ShardArgs* sh = nullptr);
uint32_t quote_parity(Ctx* c, const uint8_t* dev_bytes, uint64_t n);
// stream.cu: batches of whole records (cpb_stream_*)
struct Stream;
void stream_cut(Ctx* c, const uint8_t* in, uint64_t n, const cpb_reader_opts& o, uint64_t* cut_dev);  // enqueued, 8 bytes
Stream* stream_open(Ctx* c, const cpb_reader_opts& o, std::vector<std::pair<std::string, int>> spec, const cpb_pred* filter);
void stream_push(Stream* s, const void* bytes, uint64_t n, bool is_last);
Parsed stream_next(Stream* s, bool* done);  // table null: no complete record yet
void stream_free(Stream* s);
Ctx* stream_ctx(Stream* s);
// gather.cu
void exclusive_scan_u32(Ctx* c, const uint32_t* in, uint32_t* out, uint64_t n, uint64_t* total_dev);  // out[n] = total
// compaction of 0/1 flags into the ascending list of the set positions, in two calls so that the caller allocates the
// output in between: scan_flags scans the flags and reads the count back (one host synchronisation); compact_flags
// writes out[j] = (j-th set position) + add and the sentinel out[count] = n + add, so out holds count + 1 entries
struct FlagScan { const uint32_t* flags; uint64_t n; Buf pos; uint64_t count; };  // pos: uint32[n + 1] exclusive scan
FlagScan scan_flags(Ctx* c, const uint32_t* flags, uint64_t n);
void compact_flags(Ctx* c, const FlagScan& s, uint32_t add, uint32_t* out);
// rows row_ids[0, nout) of t (rows 0..nout-1 when row_ids is null: a view compacted into buffers of its own)
std::shared_ptr<Table> gather_rows(Ctx* c, const Table& t, const uint32_t* row_ids, int64_t nout);
// the rows of t whose flag (uint32 0/1, one per row) is set: scan_flags, compact_flags timed as compact_ids, gather_rows.
// first, when given: the position of the first set flag (one more host synchronisation when there is one)
std::shared_ptr<Table> rows_where(Ctx* c, const Table& t, const uint32_t* flags, uint64_t* first = nullptr);
std::shared_ptr<Table> filter_table(Ctx* c, const Table& t, const cpb_pred* pred);
int64_t first_false_row(Ctx* c, const Table& t, const cpb_pred* pred);
struct Compiled;  // pred.cuh
// The parse of a predicate with set terms (has_set_terms, pred.cuh): p is the unfiltered parse; its rows are filtered with
// the predicate compiled against its columns (the output columns), reusing *comp when it was compiled against the same
// names (a stream compiles once and builds its set indexes once).  The error and record counts stay the parse's; row 0's
// line is the line of the first row kept.
void filter_parsed(Ctx* c, Parsed& p, const cpb_pred* pred, std::shared_ptr<Compiled>& comp);
// rows `ids` (positions in `order`) of the index restricted to columns `cols` (row-slot path when it pays, else gather_rows)
std::shared_ptr<Table> gather_index_rows(Ctx* c, Index& ix, const std::vector<int>& cols, const uint32_t* ids, int64_t nout,
                                         RowOrder order);
std::shared_ptr<Table> concat_tables(Ctx* c, const std::vector<const Table*>& parts);
// full-key join against ix.derived.rowhash: payload columns `cols` (source column numbers, a non-empty subset of its cols)
// for every probe row, empty where the row finds no key; *matches = probe rows that found their key.  One random access
// and one host synchronisation.
std::shared_ptr<Table> rowhash_gather(Ctx* c, Index& ix, const Table& probe, const std::vector<int>& pidx, const std::vector<int>& cols,
                                      uint64_t* matches);
// sort.cu.  A missing key column (of a non-empty table) or a duplicate key of a unique index throws DataError.
std::shared_ptr<Index> build_index(Ctx* c, std::shared_ptr<Table> t, const std::vector<std::string>& keys, bool unique);
std::shared_ptr<Table> sorted_table(Ctx* c, Index& ix);  // materialises ix.table on first use
void ensure_sorted(Ctx* c, Index& ix);                    // sorts a lazily-sorted unique index on first need of the order
constexpr int MAXKEYS = 16;
constexpr uint32_t MAX_KEY_IMAGE_BYTES = 4096;  // the longest key image of an index row
struct KeyDesc {  // key columns + the widths of the order-preserving image (sort.cu)
    int nkeys;
    const uint32_t* off[MAXKEYS];
    const uint8_t* data[MAXKEYS];
    uint32_t width[MAXKEYS];     // bytes of value kept
    uint32_t lenbytes[MAXKEYS];  // bytes of the big-endian length field
    uint32_t words;              // image words per row
};
// bytes of the big-endian length field after a key column of `width` value bytes in the key image
inline uint32_t len_field_bytes(uint32_t width) { return width < 255 ? 1 : (width < 65535 ? 2 : 4); }
void describe_keys(Ctx* c, const Table& t, const std::vector<int>& kidx, const std::vector<uint32_t>& width, KeyDesc& kd);
uint32_t prefix_bytes(const Index& ix, int nk);  // image bytes covered by the first nk key columns
// head[i] = 1 when the first pbytes image bytes of row i differ from those of row i - 1 (row 0 always)
void head_flags(Ctx* c, const uint64_t* image, uint64_t n, uint32_t pbytes, uint32_t* head);
Buf pack_with_widths(Ctx* c, const Table& t, const std::vector<int>& kidx, const std::vector<uint32_t>& width, uint32_t* words_out);
// join.cu.  A join column missing from a non-empty probe table throws DataError.
std::shared_ptr<Table> join_tables(Ctx* c, const Table& probe, Index& ix, const std::vector<std::string>& cols, bool anti);
// flag[i] (uint32 0/1) = whether the key of probe row i on the probe columns pidx (the first pidx.size() key columns of
// ix) is in the index (hit) / is not (!hit): Except's test, and the set terms of a predicate.  A probe value longer than
// the index column's widest value is not in it.
Buf key_flags(Ctx* c, const Table& probe, const std::vector<int>& pidx, Index& ix, bool hit);
void find_range(Ctx* c, Index& ix, const std::vector<std::string>& values, int64_t* lo, int64_t* hi);
bool index_has_duplicates(Ctx* c, Index& ix);  // full-key probe table over the source order + self probe
// fills ix.derived.rowhash (cols set by the caller) from ix.src.  built: the table is complete; duplicate: some key occurs twice;
// overflow: some region received more keys than it can hold (no duplicate was seen, but the table is unusable)
enum class RhBuild { built, duplicate, overflow };
RhBuild rowhash_build(Ctx* c, Index& ix);
void index_dup_groups(Ctx* c, Index& ix, std::vector<int64_t>& lo, std::vector<int64_t>& hi);
void index_dedup_apply(Ctx* c, Index& ix, const std::vector<int64_t>& keep, bool bug_compatible, const Table* repl = nullptr);
// the index takes the rows of nt in their stored order: key columns, widths and key image are rebuilt from them, in_order
// is set from the image (sort.cu)
void index_adopt_rows(Ctx* c, Index& ix, std::shared_ptr<Table> nt);
// gob.cu: Index.WriteTo / LoadIndex.  gob_prefix: the file's bytes before the first row, *total = the file's size;
// gob_rows: rows [lo, hi) of the stored rows (room as table_to_csv); gob_load: an index from a whole file's bytes
std::string gob_prefix(Ctx* c, Index& ix, uint64_t* total);
Buf gob_rows(Ctx* c, Index& ix, uint64_t lo, uint64_t hi, uint64_t room, uint64_t* nbytes);
std::shared_ptr<Index> gob_load(Ctx* c, const uint8_t* bytes, uint64_t nbytes, std::vector<std::string>* key_cols);
// write.cu: ToCsv of columns cols under the header line of names (when with_header).  room: the most bytes the caller can
// take; when *nbytes exceeds it, null is returned after the length pass, before any output is allocated or written.
Buf table_to_csv(Ctx* c, const Table& t, const std::vector<int>& cols, const std::vector<std::string>& names, bool with_header,
                 uint64_t room, uint64_t* nbytes);
// json.cu: ToJSON of every column (keys in bytewise order); '[' before the first row when first, ']' appended when last;
// room as table_to_csv
Buf table_to_json(Ctx* c, const Table& t, bool first, bool last, uint64_t room, uint64_t* nbytes);
// numeric.cu: strconv.Atoi / ParseFloat(s, 64) of every row of column `col` into device values (+ nullable status)
struct NumResult {
    uint64_t nbad = 0, nrare = 0;  // failing rows, rows the exact (rare) path converted
    uint64_t first_row = 0;        // lowest failing row, its status and (up to 480 of) its bytes
    int first_status = 0;
    std::string first_value;
};
NumResult column_as_number(Ctx* c, const Table& t, int col, bool is_float, void* values, uint8_t* status);
// format.cu: computed columns.  t with column `name` set (replaced in place, else appended; the other columns share t's
// buffers) to strconv.FormatInt(v, 10) / FormatFloat(x, fmt, prec, 64) of the n device values, or to one literal value
std::shared_ptr<Table> table_set_values(Ctx* c, const Table& t, const std::string& name, const void* values, bool is_float, char fmt, int prec);
std::shared_ptr<Table> table_set_literal(Ctx* c, const Table& t, const std::string& name, const std::string& value);
// the rows of t whose keep byte is nonzero, in order
std::shared_ptr<Table> table_filter_mask(Ctx* c, const Table& t, const uint8_t* keep);

}  // namespace cpb

extern "C" void cpb_comm_release(cpb::Ctx* c);  // comm.cu

// opaque handle layouts of the C ABI
struct cpb_ctx { cpb::Ctx c; };
struct cpb_table { std::shared_ptr<cpb::Table> t; };
struct cpb_index { std::shared_ptr<cpb::Index> ix; };
struct cpb_stream { cpb::Stream* s; };

namespace cpb {
template <class F> int guarded(cpb_ctx* h, cpb_error* err, F&& body) { return guarded(h ? &h->c : nullptr, err, body); }
}  // namespace cpb
