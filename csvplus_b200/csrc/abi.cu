// abi.cu — the extern "C" boundary (include/csvplus_b200.h): context, staging memory, table
// accessors and the thin argument marshalling around the kernels in parse/gather/sort/join/write.cu.
#include <algorithm>
#include <new>

#include "core.hpp"

using namespace cpb;


namespace cpb {

std::string go_quote(const std::string& s) {
    std::string r = "\"";
    for (unsigned char ch : s) {
        if (ch == '"' || ch == '\\') { r += '\\'; r += (char)ch; }
        else if (ch == '\n') r += "\\n";
        else if (ch == '\r') r += "\\r";
        else if (ch == '\t') r += "\\t";
        else if (ch < 0x20 || ch == 0x7f) { char b[8]; snprintf(b, sizeof b, "\\x%02x", ch); r += b; }
        else r += (char)ch;
    }
    return r + "\"";
}

// Requests are rounded up to size classes (1/8 steps of the enclosing power of two, <= 12.5 % slack): batches of
// slightly different sizes then ask the stream-ordered pool for identical blocks and reuse them instead of
// mapping fresh physical memory (which costs tens of milliseconds per GB).
static size_t size_class(size_t b) {
    if (b < (1u << 20)) return (b + 511) & ~(size_t)511;
    size_t p = 1;
    while ((p << 1) <= b) p <<= 1;
    const size_t step = p >> 3;
    return (b + step - 1) / step * step;
}
DevBuf::DevBuf(Ctx* c, size_t bytes) : ctx(c), n(bytes) {
    cudaError_t e = cudaMallocAsync(&p, size_class(bytes), c->pool, c->stream);
    if (e != cudaSuccess) { cudaGetLastError(); throw CudaFail{e, "cudaMallocAsync", __FILE__, __LINE__}; }
}
DevBuf::DevBuf(Ctx* owner, Ctx* user, size_t bytes) : ctx(owner), n(bytes) {
    cudaError_t e = cudaMallocAsync(&p, size_class(bytes), owner->pool, user->stream);
    if (e != cudaSuccess) { cudaGetLastError(); throw CudaFail{e, "cudaMallocAsync", __FILE__, __LINE__}; }
}
DevBuf::~DevBuf() {
    if (p && ctx) { cudaSetDevice(ctx->device); cudaFreeAsync(p, ctx->stream); }
}

void* Ctx::pinned_scratch(size_t n) {
    if (n > pinned_n) {
        if (pinned) { cudaStreamSynchronize(stream); cudaFreeHost(pinned); pinned = nullptr; }
        size_t want = std::max<size_t>(n, 1 << 20);
        CPB_CUDA(cudaMallocHost(&pinned, want));
        pinned_n = want;
    }
    return pinned;
}

// Timing events are recycled: a step launches ~60 timed kernels, and creating / keeping thousands of live events
// over many steps is not free.  harvest() folds the records whose kernels have already finished into the stats
// without blocking; drain_events() waits for the rest.
static void fold_event(Ctx* c, PendingEvent& pe) {
    float ms = 0;
    cudaEventElapsedTime(&ms, pe.a, pe.b);
    KStat& s = c->stats[pe.name];
    s.ms += ms; s.bytes += pe.bytes;
    c->event_pool.push_back(pe.a); c->event_pool.push_back(pe.b);
}
void Ctx::harvest_events() {
    size_t done = 0;
    while (done < pending.size() && cudaEventQuery(pending[done].b) == cudaSuccess) { fold_event(this, pending[done]); done++; }
    cudaGetLastError();  // cudaErrorNotReady of the first unfinished record
    if (done) pending.erase(pending.begin(), pending.begin() + (long)done);
}
void Ctx::drain_events() {
    for (auto& pe : pending) {
        cudaEventSynchronize(pe.b);
        fold_event(this, pe);
    }
    pending.clear();
}
static cudaEvent_t take_event(Ctx* c) {
    if (!c->event_pool.empty()) { cudaEvent_t e = c->event_pool.back(); c->event_pool.pop_back(); return e; }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
}

KernelTimer::KernelTimer(Ctx* ctx, const char* nm, uint64_t algo_bytes, int launches)
    : c(ctx), on(ctx->stats_on), name(nm), bytes(algo_bytes), nlaunch(launches) {
    c->launches += launches;
    if (on) {
        if (c->pending.size() >= 64) c->harvest_events();
        a = take_event(c); b = take_event(c);
        cudaEventRecord(a, c->stream);
    }
}
KernelTimer::~KernelTimer() {
    if (on) {
        cudaEventRecord(b, c->stream);
        c->stats[name].launches += nlaunch;
        c->pending.push_back(PendingEvent{name, a, b, bytes});
    }
}

// a data error of the reference: CPB_ERR_DATA, with the error in *err
static int data_error(cpb_error* err, const DataError& d) {
    fill_error(err, d.kind, d.column_index, d.line, d.has_line, d.msg);
    return CPB_ERR_DATA;
}

int translate_exception(Ctx* c, cpb_error* err) {
    try { throw; }
    catch (const CudaFail& f) {
        char buf[400];
        snprintf(buf, sizeof buf, "CUDA error %d (%s) at %s:%d: %s", (int)f.e, cudaGetErrorString(f.e), f.file, f.line, f.what);
        if (c) c->last_error = buf;
        fill_error(err, CPB_E_CUDA, -1, 0, false, buf);
        cudaGetLastError();
        return CPB_ERR_CUDA;
    } catch (const DataError& d) {
        if (c) c->last_error = d.msg;
        return data_error(err, d);
    } catch (const ArgError& a) {
        if (c) c->last_error = a.msg;
        fill_error(err, a.status == CPB_ERR_UNSUPPORTED ? CPB_E_UNSUPPORTED : CPB_E_NONE, -1, 0, false, a.msg);
        return a.status;
    } catch (const std::bad_alloc&) {
        if (c) c->last_error = "out of host memory";
        return CPB_ERR_NOMEM;
    } catch (const std::exception& e) {
        if (c) c->last_error = e.what();
        fill_error(err, CPB_E_NONE, -1, 0, false, e.what());
        return CPB_ERR_ARG;
    } catch (...) {
        if (c) c->last_error = "unknown error";
        return CPB_ERR_ARG;
    }
}

}  // namespace cpb

static std::vector<std::string> str_list(const cpb_str* s, int n) {
    need(n <= 0 || s, "null string list");
    std::vector<std::string> v;
    for (int i = 0; i < n; i++) v.push_back(to_string(s[i]));
    return v;
}
static cpb_table* wrap(std::shared_ptr<Table> t) { return new cpb_table{std::move(t)}; }

// the table behind a handle the caller must pass
static const Table& table_of(const cpb_table* t) {
    need(t, "null table");
    return *t->t;
}
static Index& index_of(const cpb_index* ix) {
    need(ix, "null index");
    return *ix->ix;
}

// ------------------------------------------------------------------ ToCsv / ToJSON / index file output
// Where a serialiser's bytes go.  pinned: new pinned host memory, returned in *bytes; into: caller-owned (ideally
// pinned) host memory of cap bytes at host_dst; device: new device memory, returned in *bytes.
struct Dest {
    enum Mode { pinned, into, device } mode;
    void** bytes; void* host_dst; uint64_t cap;
    void check() const { need(mode == into ? !cap || host_dst : bytes != nullptr, "null destination"); }
    uint64_t limit() const { return mode == into ? cap : UINT64_MAX; }  // the most bytes the serialiser may produce
};
static void deliver(Ctx* c, const Buf& out, uint64_t total, const Dest& d, const char* too_small) {
    if (d.mode == Dest::pinned) {
        void* hp = nullptr;
        CPB_CUDA(cudaMallocHost(&hp, total ? total : 1));
        if (total) CPB_CUDA(cudaMemcpyAsync(hp, out->p, total, cudaMemcpyDeviceToHost, c->stream));
        sync_stream(c);
        *d.bytes = hp;
    } else if (d.mode == Dest::into) {
        if (total > d.cap) throw ArgError{CPB_ERR_ARG, too_small};
        if (total) {
            KernelTimer kt(c, "d2h_output", total, 0);
            CPB_CUDA(cudaMemcpyAsync(d.host_dst, out->p, total, cudaMemcpyDeviceToHost, c->stream));
        }
        sync_stream(c);
    } else {
        void* dp = nullptr;
        CPB_CUDA(cudaMallocAsync(&dp, total + 16, c->pool, c->stream));
        if (total) CPB_CUDA(cudaMemcpyAsync(dp, out->p, total, cudaMemcpyDeviceToDevice, c->stream));
        *d.bytes = dp;
    }
}
// One serialiser call: produce(c, room, &total) returns the bytes on the device, or null after its length pass when
// total exceeds room.  *nbytes = total either way; a destination that is too small gets nothing and the call fails with
// CPB_ERR_ARG (too_small).
template <class F> static int serialise(cpb_ctx* h, cpb_error* err, const Dest& d, uint64_t* nbytes, const char* too_small, F&& produce) {
    return guarded(h, err, [&](Ctx* c) {
        need(nbytes, "null nbytes");
        d.check();
        uint64_t total = 0;
        Buf out = produce(c, d.limit(), &total);
        *nbytes = total;
        deliver(c, out, total, d, too_small);
        return CPB_OK;
    });
}

// *out = make(c, t's table): the entries that derive one table from another (views and computed columns)
template <class F> static int derived_table(cpb_ctx* h, const cpb_table* t, cpb_table** out, cpb_error* err, F&& make) {
    return guarded(h, err, [&](Ctx* c) {
        const Table& T = table_of(t);
        need(out, "null out");
        *out = wrap(make(c, T));
        return CPB_OK;
    });
}

extern "C" {

int cpb_abi_version(void) { return CPB_ABI_VERSION; }

int cpb_init(int device, cpb_ctx** out) {
    if (!out) return CPB_ERR_ARG;
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || device < 0 || device >= ndev) { cudaGetLastError(); return CPB_ERR_CUDA; }  // no CPU fallback
    cpb_ctx* h = new (std::nothrow) cpb_ctx();
    if (!h) return CPB_ERR_NOMEM;
    Ctx* c = &h->c;
    try {
        c->device = device;
        CPB_CUDA(cudaSetDevice(device));
        // CPB_BLOCKING_SYNC=1: host waits sleep on an interrupt instead of spinning.  One process per GPU on a shared host:
        // N spinning ranks (+ NCCL's proxy threads) can run a cgroup into its CPU quota, and a throttled rank stalls all
        // the others at the next collective.
        if (const char* bs = getenv("CPB_BLOCKING_SYNC")) {
            if (bs[0] == '1') { cudaSetDeviceFlags(cudaDeviceScheduleBlockingSync); cudaGetLastError(); }
        }
        cudaDeviceProp prop;
        CPB_CUDA(cudaGetDeviceProperties(&prop, device));
        // sm_90a code runs on compute capability 9.0 only (the "a" features do not carry forward)
        if (prop.major != 9 || prop.minor != 0)
            throw ArgError{CPB_ERR_UNSUPPORTED, "csvplus_b200 kernels are built for sm_90a (H100) only"};
        c->sm_count = prop.multiProcessorCount;
        c->smem_optin = prop.sharedMemPerBlockOptin;
        CPB_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
        // a private stream-ordered pool per ctx: contexts running on different streams never wait on each other's
        // frees (the shared default pool may insert cross-stream dependencies to recycle memory)
        if (getenv("CPB_SHARED_POOL")) {
            CPB_CUDA(cudaDeviceGetDefaultMemPool(&c->pool, device));
        } else {
            cudaMemPoolProps props{};
            props.allocType = cudaMemAllocationTypePinned;
            props.handleTypes = cudaMemHandleTypeNone;
            props.location.type = cudaMemLocationTypeDevice;
            props.location.id = device;
            CPB_CUDA(cudaMemPoolCreate(&c->pool, &props));
            c->own_pool = true;
        }
        uint64_t thr = UINT64_MAX;  // keep freed blocks cached in the pool
        CPB_CUDA(cudaMemPoolSetAttribute(c->pool, cudaMemPoolAttrReleaseThreshold, &thr));
    } catch (...) {
        int st = translate_exception(c, nullptr);
        delete h;
        return st;
    }
    *out = h;
    return CPB_OK;
}

void cpb_shutdown(cpb_ctx* h) {
    if (!h) return;
    Ctx* c = &h->c;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    c->drain_events();
    for (cudaEvent_t e : c->event_pool) cudaEventDestroy(e);
    c->event_pool.clear();
    cpb_comm_release(c);
    if (c->pinned) cudaFreeHost(c->pinned);
    cudaStreamDestroy(c->stream);
    if (c->own_pool) cudaMemPoolDestroy(c->pool);
    delete h;
}

void* cpb_ctx_stream(cpb_ctx* h) { return h ? (void*)h->c.stream : nullptr; }
const char* cpb_last_error(cpb_ctx* h) { return h ? h->c.last_error.c_str() : ""; }

int cpb_sync(cpb_ctx* h) {
    return guarded(h, nullptr, [&](Ctx* c) {
        sync_stream(c);
        return CPB_OK;
    });
}

int cpb_pool_reserve(cpb_ctx* h, uint64_t nbytes) {
    return guarded(h, nullptr, [&](Ctx* c) {
        if (nbytes == 0) return CPB_OK;
        void* p = nullptr;
        CPB_CUDA(cudaMallocAsync(&p, nbytes, c->pool, c->stream));
        CPB_CUDA(cudaFreeAsync(p, c->stream));
        sync_stream(c);
        return CPB_OK;
    });
}

int cpb_pool_used_high(cpb_ctx* h, int reset, uint64_t* bytes) {
    return guarded(h, nullptr, [&](Ctx* c) {
        need(bytes, "null bytes");
        uint64_t v = 0;  // the attribute is a cuuint64_t (64-bit unsigned)
        if (reset) CPB_CUDA(cudaMemPoolSetAttribute(c->pool, cudaMemPoolAttrUsedMemHigh, &v));
        CPB_CUDA(cudaMemPoolGetAttribute(c->pool, cudaMemPoolAttrUsedMemHigh, &v));
        *bytes = (uint64_t)v;
        return CPB_OK;
    });
}

int cpb_host_alloc(cpb_ctx* h, uint64_t n, void** out) {
    return guarded(h, nullptr, [&](Ctx*) {
        need(out, "null out");
        CPB_CUDA(cudaMallocHost(out, n ? n : 1));
        return CPB_OK;
    });
}
int cpb_host_free(cpb_ctx* h, void* p) {
    return guarded(h, nullptr, [&](Ctx* c) {
        sync_stream(c);
        CPB_CUDA(cudaFreeHost(p));
        return CPB_OK;
    });
}
int cpb_device_alloc(cpb_ctx* h, uint64_t n, void** out) {
    return guarded(h, nullptr, [&](Ctx* c) {
        need(out, "null out");
        uint64_t padded = ((n + 15) & ~15ull) + 256;
        CPB_CUDA(cudaMallocAsync(out, padded, c->pool, c->stream));
        CPB_CUDA(cudaMemsetAsync((uint8_t*)*out + (n & ~15ull), 0, padded - (n & ~15ull), c->stream));
        return CPB_OK;
    });
}
int cpb_device_free(cpb_ctx* h, void* p) {
    return guarded(h, nullptr, [&](Ctx* c) {
        if (p) CPB_CUDA(cudaFreeAsync(p, c->stream));
        return CPB_OK;
    });
}
static int copy_sync(cpb_ctx* h, void* dst, const void* src, uint64_t n, cudaMemcpyKind kind) {
    return guarded(h, nullptr, [&](Ctx* c) {
        need(!n || (dst && src), "null copy source or destination");
        CPB_CUDA(cudaMemcpyAsync(dst, src, n, kind, c->stream));
        sync_stream(c);
        return CPB_OK;
    });
}
int cpb_memcpy_h2d(cpb_ctx* h, void* dst, const void* src, uint64_t n) { return copy_sync(h, dst, src, n, cudaMemcpyHostToDevice); }
int cpb_memcpy_d2h(cpb_ctx* h, void* dst, const void* src, uint64_t n) { return copy_sync(h, dst, src, n, cudaMemcpyDeviceToHost); }

// ------------------------------------------------------------------ parse
// host input is copied into a device buffer (32 MiB size classes: batches reuse pool blocks) followed by at least 16 zero
// bytes; device input is used in place
static const uint8_t* stage_input(Ctx* c, const void* bytes, uint64_t nbytes, int on_device, Buf& staged) {
    need(!nbytes || bytes, "null input bytes");
    if (on_device) return (const uint8_t*)bytes;
    staged = dev_alloc(c, (nbytes + 32 + (32u << 20) - 1) / (32u << 20) * (32u << 20));  // holds the zeroed 32 bytes too
    CPB_CUDA(cudaMemsetAsync(staged->as<uint8_t>() + (nbytes & ~15ull), 0, 32, c->stream));
    if (nbytes) {
        KernelTimer kt(c, "h2d_input", nbytes, 0);
        CPB_CUDA(cudaMemcpyAsync(staged->p, bytes, nbytes, cudaMemcpyHostToDevice, c->stream));
    }
    return staged->as<uint8_t>();
}
// the (name, index) pairs of a reader's header spec; a name given twice is an error (csvplus.go:1047-1049)
static std::vector<std::pair<std::string, int>> header_spec(const cpb_header_col* spec, int nspec) {
    need(nspec >= 0 && (nspec == 0 || spec), "bad header spec");
    std::vector<std::pair<std::string, int>> sp;
    for (int i = 0; i < nspec; i++) {
        std::string nm = to_string(spec[i].name);
        for (auto& s : sp) if (s.first == nm) throw ArgError{CPB_ERR_ARG, "header spec: duplicate column name: " + nm};
        sp.emplace_back(nm, spec[i].index);
    }
    return sp;
}

int cpb_parse_csv(cpb_ctx* h, const void* bytes, uint64_t nbytes, int on_device, const cpb_reader_opts* opts,
                  const cpb_header_col* spec, int nspec, const cpb_pred* filter, cpb_table** out, cpb_error* err) {
    return guarded(h, err, [&](Ctx* c) {
        need(out && opts, "null out or opts");
        *out = nullptr;
        auto sp = header_spec(spec, nspec);
        Buf staged;
        const uint8_t* dev = stage_input(c, bytes, nbytes, on_device, staged);
        const Parsed p = parse_csv(c, dev, nbytes, *opts, sp, filter, opts->header_from_first_row ? 2 : 1);
        *out = wrap(p.table);
        return p.error ? data_error(err, *p.error) : CPB_OK;
    });
}

// ------------------------------------------------------------------ streamed input (stream.cu)
int cpb_stream_open(cpb_ctx* h, const cpb_reader_opts* opts, const cpb_header_col* spec, int nspec, const cpb_pred* filter,
                    cpb_stream** out, cpb_error* err) {
    return guarded(h, err, [&](Ctx* c) {
        need(out && opts, "null out or opts");
        *out = nullptr;
        *out = new cpb_stream{stream_open(c, *opts, header_spec(spec, nspec), filter)};
        return CPB_OK;
    });
}
int cpb_stream_push(cpb_stream* st, const void* bytes, uint64_t nbytes, int is_last) {
    return guarded(st ? stream_ctx(st->s) : nullptr, nullptr, [&](Ctx*) {
        need(!nbytes || bytes, "null input bytes");
        stream_push(st->s, bytes, nbytes, is_last != 0);
        return CPB_OK;
    });
}
int cpb_stream_next(cpb_stream* st, cpb_table** out, int* done, cpb_error* err) {
    return guarded(st ? stream_ctx(st->s) : nullptr, err, [&](Ctx*) {
        need(out && done, "null out or done");
        *out = nullptr; *done = 0;
        bool fin = false;
        const Parsed p = stream_next(st->s, &fin);
        *done = fin ? 1 : 0;
        if (p.table) *out = wrap(p.table);
        return p.error ? data_error(err, *p.error) : CPB_OK;
    });
}
void cpb_stream_free(cpb_stream* st) {
    if (!st) return;
    Ctx* c = stream_ctx(st->s); DeviceGuard g(c);
    stream_free(st->s);
    delete st;
}

// ------------------------------------------------------------------ byte-range shards of one file (SURVEY §8e)
// the input of the shard helpers on the device: they read 16 bytes at a time
static const uint8_t* stage_aligned(Ctx* c, const void* bytes, uint64_t nbytes, int on_device, Buf& staged) {
    const uint8_t* dev = stage_input(c, bytes, nbytes, on_device, staged);
    need((reinterpret_cast<uintptr_t>(dev) & 15) == 0, "device input must be 16-byte aligned");
    return dev;
}
int cpb_csv_quote_parity(cpb_ctx* h, const void* bytes, uint64_t nbytes, int on_device, uint32_t* parity) {
    return guarded(h, nullptr, [&](Ctx* c) {
        need(parity, "null parity");
        Buf staged;
        *parity = quote_parity(c, stage_aligned(c, bytes, nbytes, on_device, staged), nbytes);
        return CPB_OK;
    });
}
int cpb_csv_stream_cut(cpb_ctx* h, const void* bytes, uint64_t nbytes, int on_device, const cpb_reader_opts* opts, uint64_t* cut) {
    return guarded(h, nullptr, [&](Ctx* c) {
        need(cut && opts, "null cut or opts");
        Buf staged;
        const uint8_t* dev = stage_aligned(c, bytes, nbytes, on_device, staged);
        Buf out = dev_alloc(c, 16);
        stream_cut(c, dev, nbytes, *opts, out->as<uint64_t>());
        *cut = read_back<uint64_t>(c, out->p);
        return CPB_OK;
    });
}
int cpb_parse_csv_shard(cpb_ctx* h, const void* bytes, uint64_t nbytes, int on_device, uint64_t own_bytes, int shard_index, int is_last,
                        uint32_t initial_parity, const cpb_reader_opts* opts, const cpb_header_col* spec, int nspec, const cpb_pred* filter,
                        cpb_table** out, uint64_t* records, cpb_error* err) {
    return guarded(h, err, [&](Ctx* c) -> int {
        need(out && opts, "null out or opts");
        need(shard_index >= 0 && nspec >= 0 && (nspec == 0 || spec), "bad shard index or header spec");
        *out = nullptr;
        std::vector<std::pair<std::string, int>> sp;
        for (int i = 0; i < nspec; i++) sp.emplace_back(to_string(spec[i].name), spec[i].index);
        Buf staged;
        const uint8_t* dev = stage_input(c, bytes, nbytes, on_device, staged);
        const uint64_t base = opts->header_from_first_row ? 2 : 1;
        const ShardArgs sh{own_bytes, shard_index, is_last != 0, initial_parity};
        const Parsed p = parse_csv(c, dev, nbytes, *opts, sp, filter, base, &sh);
        if (records) *records = p.records;
        *out = wrap(p.table);
        if (!p.error) return CPB_OK;
        // the line is LOCAL: (0-based) ordinal of the failing record among this shard's records; the host adds the records
        // of the shards before it and the reader's base (csvplus.go:1102-1137)
        DataError local = *p.error;
        local.line = local.line >= base ? local.line - base : 0;
        return data_error(err, local);
    });
}

// ------------------------------------------------------------------ tables
int64_t cpb_table_num_rows(const cpb_table* t) { return t ? t->t->nrows : -1; }
int cpb_table_num_cols(const cpb_table* t) { return t ? (int)t->t->cols.size() : -1; }
int cpb_table_col_name(const cpb_table* t, int col, cpb_str* out) {
    if (!t || !out || col < 0 || col >= (int)t->t->cols.size()) return CPB_ERR_ARG;
    out->ptr = t->t->cols[col].name.data(); out->len = t->t->cols[col].name.size();
    return CPB_OK;
}
int cpb_table_find_col(const cpb_table* t, cpb_str name) { return t ? t->t->find(to_string(name)) : -1; }
int cpb_table_col_field(const cpb_table* t, int col) {
    if (!t || col < 0 || col >= (int)t->t->src_field.size()) return -1;
    return t->t->src_field[col];
}
int cpb_table_record_fields(const cpb_table* t) { return t ? t->t->record_fields : -1; }

static void need_rows(const Table& T, int col, int64_t lo, int64_t hi) {
    if (col < 0 || col >= (int)T.cols.size() || lo < 0 || hi < lo || hi > T.nrows) throw ArgError{CPB_ERR_ARG, "bad column/row range"};
}

int cpb_table_col_bytes(cpb_ctx* h, const cpb_table* t, int col, int64_t lo, int64_t hi, uint64_t* nbytes) {
    return guarded(h, nullptr, [&](Ctx* c) {
        const Table& T = table_of(t);
        need(nbytes, "null nbytes");
        need_rows(T, col, lo, hi);
        uint32_t e[2];
        CPB_CUDA(cudaMemcpyAsync(&e[0], T.cols[col].off() + lo, 4, cudaMemcpyDeviceToHost, c->stream));
        CPB_CUDA(cudaMemcpyAsync(&e[1], T.cols[col].off() + hi, 4, cudaMemcpyDeviceToHost, c->stream));
        sync_stream(c);
        *nbytes = e[1] - e[0];
        return CPB_OK;
    });
}

int cpb_table_fetch_column(cpb_ctx* h, const cpb_table* t, int col, int64_t lo, int64_t hi, int64_t* offsets_out,
                           uint8_t* data_out, uint64_t cap) {
    return guarded(h, nullptr, [&](Ctx* c) {
        const Table& T = table_of(t);
        need_rows(T, col, lo, hi);
        size_t cnt = (size_t)(hi - lo) + 1;
        std::vector<uint32_t> tmp(cnt);
        CPB_CUDA(cudaMemcpyAsync(tmp.data(), T.cols[col].off() + lo, cnt * 4, cudaMemcpyDeviceToHost, c->stream));
        sync_stream(c);
        uint64_t total = tmp[cnt - 1] - tmp[0];
        if (offsets_out) for (size_t i = 0; i < cnt; i++) offsets_out[i] = (int64_t)(tmp[i] - tmp[0]);
        if (data_out) {
            if (total > cap) throw ArgError{CPB_ERR_ARG, "data_out too small"};
            if (total) {
                CPB_CUDA(cudaMemcpyAsync(data_out, T.cols[col].bytes() + tmp[0], total, cudaMemcpyDeviceToHost, c->stream));
                sync_stream(c);
            }
        }
        return CPB_OK;
    });
}

int cpb_table_column_device(const cpb_table* t, int col, const uint32_t** offsets, const uint8_t** data) {
    if (!t || !offsets || !data || col < 0 || col >= (int)t->t->cols.size()) return CPB_ERR_ARG;
    *offsets = t->t->cols[col].off(); *data = t->t->cols[col].bytes();
    return CPB_OK;
}

// the arguments of a table given as ncols arrays of nrows values
static void need_columns(int ncols, const cpb_str* names, const void* offsets, const void* data, int64_t nrows, cpb_table** out) {
    need(out, "null out");
    need(nrows >= 0 && (ncols <= 0 || (names && offsets && data)), "bad column arrays");
}

int cpb_table_from_host(cpb_ctx* h, int ncols, const cpb_str* names, const int64_t* const* offsets,
                        const uint8_t* const* data, int64_t nrows, cpb_table** out) {
    return guarded(h, nullptr, [&](Ctx* c) {
        need_columns(ncols, names, offsets, data, nrows, out);
        auto t = std::make_shared<Table>(); t->ctx = c; t->nrows = nrows;
        for (int i = 0; i < ncols; i++) {
            need(offsets[i], "null column offsets");
            Column col; col.name = to_string(names[i]);
            std::vector<uint32_t> off((size_t)nrows + 1);
            for (int64_t r = 0; r <= nrows; r++) {
                int64_t v = offsets[i][r] - offsets[i][0];
                if (v < 0 || v > 0xffffffffll) throw DataError{CPB_E_TOO_LARGE, i, 0, false, "column exceeds 4 GiB"};
                off[(size_t)r] = (uint32_t)v;
            }
            col.offsets = dev_alloc(c, off.size() * 4);
            CPB_CUDA(cudaMemcpyAsync(col.offsets->p, off.data(), off.size() * 4, cudaMemcpyHostToDevice, c->stream));
            uint64_t total = off.back();
            need(!total || data[i], "null column data");
            col.data = dev_alloc(c, total + 16);
            if (total) CPB_CUDA(cudaMemcpyAsync(col.data->p, data[i] + offsets[i][0], total, cudaMemcpyHostToDevice, c->stream));
            sync_stream(c);
            t->cols.push_back(col);
        }
        *out = wrap(t);
        return CPB_OK;
    });
}

int cpb_table_from_device(cpb_ctx* h, int ncols, const cpb_str* names, const uint32_t* const* offsets,
                          const uint8_t* const* data, int64_t nrows, cpb_table** out) {
    return guarded(h, nullptr, [&](Ctx* c) {
        need_columns(ncols, names, offsets, data, nrows, out);
        // the caller's arrays are wrapped without ownership and copied by the concat path, which rebases offsets that do not
        // start at 0 (row-range views exported by cpb_table_column_device) and reads all extents with one host round trip
        Table view; view.ctx = c; view.nrows = nrows;
        for (int i = 0; i < ncols; i++) {
            need(offsets[i], "null column offsets");
            Column col; col.name = to_string(names[i]);
            col.offsets = std::make_shared<DevBuf>(DevBuf::Borrow{}, offsets[i], ((size_t)nrows + 1) * 4);
            col.data = std::make_shared<DevBuf>(DevBuf::Borrow{}, data[i], 0);
            view.cols.push_back(col);
        }
        *out = wrap(concat_tables(c, {&view}));
        return CPB_OK;
    });
}

int cpb_table_select(cpb_ctx* h, const cpb_table* t, const cpb_str* cols, int n, cpb_table** out, cpb_error* err) {
    return derived_table(h, t, out, err, [&](Ctx* c, const Table& T) {
        if (n <= 0) throw ArgError{CPB_ERR_ARG, "no columns specified in SelectColumns()"};  // csvplus.go:512-514
        auto names = str_list(cols, n);
        std::vector<int> pick;
        for (int i = 0; i < n; i++) {
            int k = T.find(names[i]);
            if (k < 0) {
                if (T.nrows == 0) { pick.clear(); break; }  // no rows => Row.Select never runs
                throw DataError{CPB_E_MISSING_COLUMN, i, T.first_line, true, "missing column " + go_quote(names[i])};  // csvplus.go:129
            }
            if (std::find(pick.begin(), pick.end(), k) == pick.end()) pick.push_back(k);  // a Go map holds a name once
        }
        auto r = table_view(c, T, 0, T.nrows, &pick); r->first_line = T.first_line;
        return r;
    });
}

int cpb_table_drop(cpb_ctx* h, const cpb_table* t, const cpb_str* cols, int n, cpb_table** out) {
    return derived_table(h, t, out, nullptr, [&](Ctx* c, const Table& T) {
        if (n <= 0) throw ArgError{CPB_ERR_ARG, "no columns specified in DropColumns()"};  // csvplus.go:494-496
        auto names = str_list(cols, n);
        std::vector<int> pick;
        for (int k = 0; k < (int)T.cols.size(); k++)
            if (std::find(names.begin(), names.end(), T.cols[k].name) == names.end()) pick.push_back(k);
        auto r = table_view(c, T, 0, T.nrows, &pick); r->first_line = T.first_line;
        return r;
    });
}

int cpb_table_slice(cpb_ctx* h, const cpb_table* t, int64_t lo, int64_t hi, cpb_table** out) {
    return derived_table(h, t, out, nullptr, [&](Ctx* c, const Table& T) {
        if (lo < 0) lo = 0;
        if (hi > T.nrows) hi = T.nrows;
        if (hi < lo) hi = lo;
        auto r = table_view(c, T, lo, hi); r->first_line = T.first_line + (uint64_t)lo;
        return r;
    });
}

int cpb_table_filter(cpb_ctx* h, const cpb_table* t, const cpb_pred* pred, cpb_table** out) {
    return derived_table(h, t, out, nullptr, [&](Ctx* c, const Table& T) { return filter_table(c, T, pred); });
}

int cpb_table_first_false(cpb_ctx* h, const cpb_table* t, const cpb_pred* pred, int64_t* row) {
    return guarded(h, nullptr, [&](Ctx* c) {
        const Table& T = table_of(t);
        need(row, "null row");
        *row = first_false_row(c, T, pred);
        return CPB_OK;
    });
}

int cpb_table_concat(cpb_ctx* h, const cpb_table* const* parts, int nparts, cpb_table** out) {
    return guarded(h, nullptr, [&](Ctx* c) {
        need(out, "null out");
        if (nparts <= 0) throw ArgError{CPB_ERR_ARG, "no parts"};
        need(parts, "null parts");
        std::vector<const Table*> ps;
        for (int i = 0; i < nparts; i++) ps.push_back(&table_of(parts[i]));
        *out = wrap(concat_tables(c, ps));
        return CPB_OK;
    });
}

void cpb_table_free(cpb_table* t) {
    if (!t) return;
    if (t->t && t->t->ctx) { std::unique_lock<std::mutex> lk(t->t->ctx->mu); cudaSetDevice(t->t->ctx->device); t->t.reset(); }
    delete t;
}

// ------------------------------------------------------------------ index / join
int cpb_index_build(cpb_ctx* h, const cpb_table* t, const cpb_str* key_cols, int nkeys, int unique, cpb_index** out,
                    cpb_error* err) {
    return guarded(h, err, [&](Ctx* c) {
        need(t && out, "null table or out");
        *out = nullptr;
        if (nkeys <= 0) throw ArgError{CPB_ERR_ARG, "empty column list in CreateIndex()"};  // csvplus.go:709-710
        auto keys = str_list(key_cols, nkeys);
        for (int i = 0; i < nkeys; i++)
            for (int j = i + 1; j < nkeys; j++)
                if (keys[i] == keys[j]) throw ArgError{CPB_ERR_ARG, "duplicate column name(s) in CreateIndex()"};  // :714-716
        *out = new cpb_index{build_index(c, t->t, keys, unique != 0)};
        return CPB_OK;
    });
}
int64_t cpb_index_num_rows(const cpb_index* ix) { return ix ? ix->ix->nrows : -1; }
int cpb_index_num_keys(const cpb_index* ix) { return ix ? (int)ix->ix->key_cols.size() : -1; }
int cpb_index_table(cpb_ctx* h, const cpb_index* ix, cpb_table** out) {
    return guarded(h, nullptr, [&](Ctx* c) {
        Index& X = index_of(ix);
        need(out, "null out");
        *out = wrap(sorted_table(c, X));
        return CPB_OK;
    });
}
// the stored rows whose leading key columns equal the n values, as a view (all of them when n is 0)
static std::shared_ptr<Table> rows_with_prefix(Ctx* c, Index& X, const cpb_str* values, int n) {
    int64_t lo = 0, hi = X.nrows;
    if (n > 0) find_range(c, X, str_list(values, n), &lo, &hi);
    return table_view(c, *sorted_table(c, X), lo, hi);
}
int cpb_index_find(cpb_ctx* h, const cpb_index* ix, const cpb_str* values, int n, cpb_table** out) {
    return guarded(h, nullptr, [&](Ctx* c) {
        Index& X = index_of(ix);
        need(out, "null out");
        if (n > (int)X.key_cols.size()) throw ArgError{CPB_ERR_ARG, "too many columns in indexImpl.find()"};  // csvplus.go:876-878
        *out = wrap(rows_with_prefix(c, X, values, n));
        return CPB_OK;
    });
}
int cpb_index_sub(cpb_ctx* h, const cpb_index* ix, const cpb_str* values, int n, cpb_index** out) {
    return guarded(h, nullptr, [&](Ctx* c) {
        Index& X = index_of(ix);
        need(out, "null out");
        if (n >= (int)X.key_cols.size()) throw ArgError{CPB_ERR_ARG, "too many values in SubIndex()"};  // csvplus.go:633-635
        // the slice in the parent's stored order, not re-sorted (csvplus.go:637-640): on a parent in key order it is already
        // sorted on the remaining key columns; on one out of key order it keeps that order, and the searches follow it
        auto view = rows_with_prefix(c, X, values, n);
        std::vector<std::string> keys(X.key_cols.begin() + (n > 0 ? n : 0), X.key_cols.end());
        if (view->nrows == 0) {  // (an empty index also from a parent whose table lacks the key columns)
            *out = new cpb_index{build_index(c, view, keys, false)};
            return CPB_OK;
        }
        auto sub = std::make_shared<Index>();
        sub->ctx = c; sub->key_cols = keys; sub->key_col_idx.assign(keys.size(), -1);
        index_adopt_rows(c, *sub, view);
        *out = new cpb_index{sub};
        return CPB_OK;
    });
}
int cpb_index_dup_groups(cpb_ctx* h, const cpb_index* ix, int64_t* ngroups, int64_t** lo, int64_t** hi) {
    return guarded(h, nullptr, [&](Ctx* c) -> int {
        Index& X = index_of(ix);
        need(ngroups && lo && hi, "null ngroups, lo or hi");
        std::vector<int64_t> a, b;
        index_dup_groups(c, X, a, b);
        *ngroups = (int64_t)a.size();
        *lo = (int64_t*)malloc((a.size() + 1) * 8); *hi = (int64_t*)malloc((a.size() + 1) * 8);
        if (!*lo || !*hi) return CPB_ERR_NOMEM;
        if (!a.empty()) { memcpy(*lo, a.data(), a.size() * 8); memcpy(*hi, b.data(), b.size() * 8); }
        return CPB_OK;
    });
}
int cpb_index_dedup_apply2(cpb_ctx* h, cpb_index* ix, int64_t ngroups, const int64_t* keep, const cpb_table* replacements,
                           int bug_compatible, cpb_error* err) {
    return guarded(h, err, [&](Ctx* c) {
        Index& X = index_of(ix);
        need(ngroups <= 0 || keep, "null keep");
        std::vector<int64_t> k(keep, keep + (ngroups > 0 ? ngroups : 0));
        index_dedup_apply(c, X, k, bug_compatible != 0, replacements ? replacements->t.get() : nullptr);
        return CPB_OK;
    });
}
int cpb_index_dedup_apply(cpb_ctx* h, cpb_index* ix, int64_t ngroups, const int64_t* keep, int bug_compatible) {
    return cpb_index_dedup_apply2(h, ix, ngroups, keep, nullptr, bug_compatible, nullptr);
}
void cpb_index_free(cpb_index* ix) {
    if (!ix) return;
    if (ix->ix && ix->ix->ctx) { std::unique_lock<std::mutex> lk(ix->ix->ctx->mu); cudaSetDevice(ix->ix->ctx->device); ix->ix.reset(); }
    delete ix;
}
void cpb_free(void* p) { free(p); }
int cpb_index_key_col(const cpb_index* ix, int k, cpb_str* out) {
    if (!ix || !out || k < 0 || k >= (int)ix->ix->key_cols.size()) return CPB_ERR_ARG;
    out->ptr = ix->ix->key_cols[k].data(); out->len = ix->ix->key_cols[k].size();
    return CPB_OK;
}

static int join_common(cpb_ctx* h, const cpb_table* probe, const cpb_index* ix, const cpb_str* cols, int n, JoinMode mode,
                       cpb_table** out, cpb_error* err) {
    return guarded(h, err, [&](Ctx* c) {
        const Table& P = table_of(probe);
        Index& X = index_of(ix);
        need(out, "null out");
        *out = nullptr;
        std::vector<std::string> names = n ? str_list(cols, n) : X.key_cols;  // natural join, csvplus.go:546-547
        if (names.size() > X.key_cols.size())  // :548-549, :591-592
            throw ArgError{CPB_ERR_ARG, mode == JoinMode::anti   ? "too many source columns in Except()"
                                        : mode == JoinMode::left ? "too many source columns in LeftJoin()"
                                                                 : "too many source columns in Join()"};
        *out = wrap(join_tables(c, P, X, names, mode));
        return CPB_OK;
    });
}
int cpb_join(cpb_ctx* h, const cpb_table* probe, const cpb_index* ix, const cpb_str* cols, int n, cpb_table** out, cpb_error* err) {
    return join_common(h, probe, ix, cols, n, JoinMode::inner, out, err);
}
int cpb_except(cpb_ctx* h, const cpb_table* probe, const cpb_index* ix, const cpb_str* cols, int n, cpb_table** out, cpb_error* err) {
    return join_common(h, probe, ix, cols, n, JoinMode::anti, out, err);
}
int cpb_left_join(cpb_ctx* h, const cpb_table* probe, const cpb_index* ix, const cpb_str* cols, int n, cpb_table** out, cpb_error* err) {
    return join_common(h, probe, ix, cols, n, JoinMode::left, out, err);
}

// ------------------------------------------------------------------ index files (gob.cu)
int cpb_index_gob_begin(cpb_ctx* h, const cpb_index* ix, void* prefix, uint64_t cap, uint64_t* prefix_len, uint64_t* total_len,
                        cpb_error* err) {
    return guarded(h, err, [&](Ctx* c) {
        Index& X = index_of(ix);
        need(prefix_len && total_len && (!cap || prefix), "null prefix, prefix_len or total_len");
        const std::string p = gob_prefix(c, X, total_len);
        *prefix_len = p.size();
        if (p.size() > cap) throw ArgError{CPB_ERR_ARG, "index file prefix destination too small"};
        memcpy(prefix, p.data(), p.size());
        return CPB_OK;
    });
}
int cpb_index_gob_into(cpb_ctx* h, const cpb_index* ix, int64_t lo, int64_t hi, void* host_dst, uint64_t cap, uint64_t* nbytes,
                       cpb_error* err) {
    return serialise(h, err, Dest{Dest::into, nullptr, host_dst, cap}, nbytes, "index file destination too small",
                     [&](Ctx* c, uint64_t room, uint64_t* total) {
        Index& X = index_of(ix);
        if (lo < 0 || hi < lo || hi > X.nrows) throw ArgError{CPB_ERR_ARG, "bad row range"};
        return gob_rows(c, X, (uint64_t)lo, (uint64_t)hi, room, total);
    });
}
int cpb_index_load_gob(cpb_ctx* h, const void* bytes, uint64_t nbytes, cpb_index** out, cpb_error* err) {
    return guarded(h, err, [&](Ctx* c) {
        need(out && (!nbytes || bytes), "null out or bytes");
        *out = nullptr;
        std::vector<std::string> keys;
        *out = new cpb_index{gob_load(c, (const uint8_t*)bytes, nbytes, &keys)};
        return CPB_OK;
    });
}

// ------------------------------------------------------------------ ToCsv
// in mode `into` the header line is written only when asked for (a csv.Writer writes it once, before the first batch:
// csvplus.go:387)
static int to_csv_common(cpb_ctx* h, const cpb_table* t, const cpb_str* cols, int n, int with_header, const Dest& d, uint64_t* nbytes,
                         cpb_error* err) {
    return serialise(h, err, d, nbytes, "ToCsv destination too small", [&](Ctx* c, uint64_t room, uint64_t* total) {
        const Table& T = table_of(t);
        if (n <= 0) throw ArgError{CPB_ERR_ARG, "empty column list in ToCsv() function"};  // csvplus.go:380-382
        auto names = str_list(cols, n);
        std::vector<int> idx;
        for (int i = 0; i < n; i++) {
            int k = T.find(names[i]);
            if (k < 0 && T.nrows > 0)
                throw DataError{CPB_E_MISSING_COLUMN, i, T.first_line, true, "missing column " + go_quote(names[i])};  // :392, :145
            idx.push_back(k);
        }
        return table_to_csv(c, T, idx, names, with_header != 0, room, total);
    });
}
int cpb_table_to_csv_into(cpb_ctx* h, const cpb_table* t, const cpb_str* cols, int n, int with_header, void* host_dst,
                          uint64_t cap, uint64_t* nbytes, cpb_error* err) {
    return to_csv_common(h, t, cols, n, with_header, Dest{Dest::into, nullptr, host_dst, cap}, nbytes, err);
}
int cpb_table_to_csv(cpb_ctx* h, const cpb_table* t, const cpb_str* cols, int n, void** bytes, uint64_t* nbytes, cpb_error* err) {
    return to_csv_common(h, t, cols, n, 1, Dest{Dest::pinned, bytes, nullptr, 0}, nbytes, err);
}
int cpb_table_to_csv_device(cpb_ctx* h, const cpb_table* t, const cpb_str* cols, int n, void** bytes, uint64_t* nbytes, cpb_error* err) {
    return to_csv_common(h, t, cols, n, 1, Dest{Dest::device, bytes, nullptr, 0}, nbytes, err);
}

// ------------------------------------------------------------------ ToJSON
static int to_json_common(cpb_ctx* h, const cpb_table* t, int first, int last, const Dest& d, uint64_t* nbytes, cpb_error* err) {
    return serialise(h, err, d, nbytes, "ToJSON destination too small", [&](Ctx* c, uint64_t room, uint64_t* total) {
        return table_to_json(c, table_of(t), first != 0, last != 0, room, total);
    });
}
int cpb_table_to_json(cpb_ctx* h, const cpb_table* t, int first_batch, int last_batch, void** bytes, uint64_t* nbytes, cpb_error* err) {
    return to_json_common(h, t, first_batch, last_batch, Dest{Dest::pinned, bytes, nullptr, 0}, nbytes, err);
}
int cpb_table_to_json_into(cpb_ctx* h, const cpb_table* t, int first_batch, int last_batch, void* host_dst, uint64_t cap,
                           uint64_t* nbytes, cpb_error* err) {
    return to_json_common(h, t, first_batch, last_batch, Dest{Dest::into, nullptr, host_dst, cap}, nbytes, err);
}
int cpb_table_to_json_device(cpb_ctx* h, const cpb_table* t, int first_batch, int last_batch, void** bytes, uint64_t* nbytes,
                             cpb_error* err) {
    return to_json_common(h, t, first_batch, last_batch, Dest{Dest::device, bytes, nullptr, 0}, nbytes, err);
}

// ------------------------------------------------------------------ numeric columns
// Row.ValueAsInt / ValueAsFloat64 (csvplus.go:163-205), and ParseFloat(s, 32) in the same closure, of every row; the
// error is the first failing row's
static int column_as_common(cpb_ctx* h, const cpb_table* t, cpb_str column, NumKind kind, void* values, uint8_t* status,
                            uint64_t* nbad, cpb_error* err) {
    return guarded(h, err, [&](Ctx* c) {
        const Table& T = table_of(t);
        need(nbad && (values || T.nrows == 0), "null nbad or values");
        *nbad = 0;
        const std::string name = to_string(column);
        const int k = T.find(name);
        if (T.nrows == 0) return CPB_OK;
        if (k < 0) throw DataError{CPB_E_MISSING_COLUMN, -1, 0, false, "missing column " + go_quote(name)};  // :170, :192
        NumResult r = column_as_number(c, T, k, kind, values, status);
        *nbad = r.nbad;
        if (r.nbad) throw number_error(name, kind, r);
        return CPB_OK;
    });
}
int cpb_table_column_as_int64(cpb_ctx* h, const cpb_table* t, cpb_str column, int64_t* values, uint8_t* status, uint64_t* nbad,
                              cpb_error* err) {
    return column_as_common(h, t, column, NumKind::Int64, values, status, nbad, err);
}
int cpb_table_column_as_float64(cpb_ctx* h, const cpb_table* t, cpb_str column, double* values, uint8_t* status, uint64_t* nbad,
                                cpb_error* err) {
    return column_as_common(h, t, column, NumKind::Float64, values, status, nbad, err);
}
int cpb_table_column_as_float32(cpb_ctx* h, const cpb_table* t, cpb_str column, float* values, uint8_t* status, uint64_t* nbad,
                                cpb_error* err) {
    return column_as_common(h, t, column, NumKind::Float32, values, status, nbad, err);
}

// ------------------------------------------------------------------ computed columns
int cpb_table_set_int64(cpb_ctx* h, const cpb_table* t, cpb_str column, const int64_t* dev_values, cpb_table** out, cpb_error* err) {
    return derived_table(h, t, out, err, [&](Ctx* c, const Table& T) {
        return table_set_values(c, T, to_string(column), dev_values, NumKind::Int64, 'f', 0);
    });
}
int cpb_table_set_float64(cpb_ctx* h, const cpb_table* t, cpb_str column, const double* dev_values, char fmt, int prec, cpb_table** out,
                          cpb_error* err) {
    return derived_table(h, t, out, err, [&](Ctx* c, const Table& T) {
        return table_set_values(c, T, to_string(column), dev_values, NumKind::Float64, fmt, prec);
    });
}
int cpb_table_set_float32(cpb_ctx* h, const cpb_table* t, cpb_str column, const float* dev_values, char fmt, int prec, cpb_table** out,
                          cpb_error* err) {
    return derived_table(h, t, out, err, [&](Ctx* c, const Table& T) {
        return table_set_values(c, T, to_string(column), dev_values, NumKind::Float32, fmt, prec);
    });
}
int cpb_table_set_literal(cpb_ctx* h, const cpb_table* t, cpb_str column, cpb_str value, cpb_table** out, cpb_error* err) {
    return derived_table(h, t, out, err, [&](Ctx* c, const Table& T) { return table_set_literal(c, T, to_string(column), to_string(value)); });
}
int cpb_table_filter_flags(cpb_ctx* h, const cpb_table* t, const uint8_t* dev_keep, cpb_table** out, cpb_error* err) {
    return derived_table(h, t, out, err, [&](Ctx* c, const Table& T) { return table_filter_mask(c, T, dev_keep); });
}

// ------------------------------------------------------------------ categorical codes
int cpb_table_column_codes(cpb_ctx* h, const cpb_table* t, cpb_str column, int64_t* dev_codes, cpb_table** dictionary, cpb_error* err) {
    return guarded(h, err, [&](Ctx* c) {
        const Table& T = table_of(t);
        need(dictionary && (dev_codes || T.nrows == 0), "null dictionary or codes");
        const std::string name = to_string(column);
        const int k = T.find(name);
        if (T.nrows == 0) {
            auto d = std::make_shared<Table>(); d->ctx = c;
            Column col = empty_column(c); col.name = name;
            d->cols.push_back(col);
            *dictionary = wrap(d);
            return CPB_OK;
        }
        if (k < 0) throw DataError{CPB_E_MISSING_COLUMN, -1, 0, false, "missing column " + go_quote(name)};  // as column_as_int64
        *dictionary = wrap(column_codes(c, T, k, dev_codes));
        return CPB_OK;
    });
}
int cpb_table_set_codes(cpb_ctx* h, const cpb_table* t, cpb_str column, const int64_t* dev_codes, const cpb_table* dictionary,
                        cpb_table** out, cpb_error* err) {
    return derived_table(h, t, out, err, [&](Ctx* c, const Table& T) {
        return table_set_codes(c, T, to_string(column), dev_codes, table_of(dictionary));
    });
}

// ------------------------------------------------------------------ GroupBy
static Groups& groups_of(Ctx* c, const cpb_groups* g) {
    need(g, "null groups");
    need(groups_ctx(*g->g) == c, "groups of another context");
    return *g->g;
}
int cpb_groups_open(cpb_ctx* h, const cpb_str* keys, int nkeys, const cpb_agg* aggs, int naggs, cpb_groups** out) {
    return guarded(h, nullptr, [&](Ctx* c) {
        need(out && (naggs <= 0 || aggs), "null out or aggregates");
        std::vector<GroupAgg> ag;
        for (int i = 0; i < naggs; i++) ag.push_back(GroupAgg{aggs[i].op, aggs[i].kind, to_string(aggs[i].column)});
        *out = new cpb_groups{groups_open(c, str_list(keys, nkeys), ag)};
        return CPB_OK;
    });
}
int cpb_groups_push(cpb_ctx* h, cpb_groups* g, const cpb_table* t, cpb_error* err) {
    return guarded(h, err, [&](Ctx* c) {
        groups_push(c, groups_of(c, g), table_of(t));
        return CPB_OK;
    });
}
int cpb_groups_result(cpb_ctx* h, const cpb_groups* g, cpb_table** keys, uint64_t* ngroups) {
    return guarded(h, nullptr, [&](Ctx* c) {
        const Groups& G = groups_of(c, g);
        need(keys && ngroups, "null keys or ngroups");
        *keys = wrap(groups_keys(c, G));
        *ngroups = groups_count(G);
        return CPB_OK;
    });
}
int cpb_groups_values(cpb_ctx* h, const cpb_groups* g, int i, void* dev_dst) {
    return guarded(h, nullptr, [&](Ctx* c) {
        groups_values(c, groups_of(c, g), i, dev_dst);
        return CPB_OK;
    });
}
int cpb_groups_free(cpb_ctx* h, cpb_groups* g) {
    return guarded(h, nullptr, [&](Ctx* c) {
        groups_of(c, g);
        groups_free(g->g);
        delete g;
        return CPB_OK;
    });
}

// ------------------------------------------------------------------ OrderBy
int cpb_table_order_by(cpb_ctx* h, const cpb_table* t, const cpb_order_key* keys, int nkeys, uint64_t limit, const cpb_table* before,
                       cpb_table** out, cpb_error* err) {
    return guarded(h, err, [&](Ctx* c) {
        const Table& T = table_of(t);
        need(out && (nkeys <= 0 || keys), "null out or keys");
        *out = nullptr;
        std::vector<OrderKey> ks;
        for (int i = 0; i < nkeys; i++) ks.push_back(OrderKey{to_string(keys[i].column), keys[i].kind, keys[i].descending != 0});
        *out = wrap(order_table(c, T, ks, limit, before ? &table_of(before) : nullptr));
        return CPB_OK;
    });
}

// ------------------------------------------------------------------ Sprintf columns and text
int cpb_table_set_sprintf(cpb_ctx* h, const cpb_table* t, cpb_str column, cpb_str format, const cpb_str* args, int nargs, cpb_table** out,
                          cpb_error* err) {
    return derived_table(h, t, out, err, [&](Ctx* c, const Table& T) {
        return table_set_sprintf(c, T, to_string(column), to_string(format), str_list(args, nargs));
    });
}
int cpb_table_sprintf_into(cpb_ctx* h, const cpb_table* t, cpb_str format, const cpb_str* args, int nargs, void* host_dst, uint64_t cap,
                           uint64_t* nbytes, cpb_error* err) {
    return serialise(h, err, Dest{Dest::into, nullptr, host_dst, cap}, nbytes, "Sprintf destination too small",
                     [&](Ctx* c, uint64_t room, uint64_t* total) {
                         return table_sprintf(c, table_of(t), to_string(format), str_list(args, nargs), room, total);
                     });
}

// ------------------------------------------------------------------ stats
int cpb_stats_enable(cpb_ctx* h, int on) {
    return guarded(h, nullptr, [&](Ctx* c) { c->stats_on = on != 0; return CPB_OK; });
}
int cpb_stats_reset(cpb_ctx* h) {
    return guarded(h, nullptr, [&](Ctx* c) {
        c->drain_events(); c->stats.clear();
        return CPB_OK;
    });
}
int cpb_stats_get(cpb_ctx* h, cpb_kstat* out, int cap, int* n) {
    return guarded(h, nullptr, [&](Ctx* c) {
        need(n && (cap <= 0 || out), "null n or out");
        c->drain_events();
        int i = 0;
        for (auto& kv : c->stats) {
            if (i < cap) {
                memset(&out[i], 0, sizeof(cpb_kstat));
                strncpy(out[i].name, kv.first.c_str(), sizeof(out[i].name) - 1);
                out[i].launches = kv.second.launches; out[i].ms = kv.second.ms; out[i].algo_bytes = kv.second.bytes;
            }
            i++;
        }
        *n = i;
        return CPB_OK;
    });
}
uint64_t cpb_kernel_launches(cpb_ctx* h) { return h ? h->c.launches : 0; }
uint64_t cpb_host_syncs(cpb_ctx* h) { return h ? h->c.host_syncs : 0; }

}  // extern "C"
