// comm.cu — the one exchange step of the multi-GPU path (SURVEY §8e): the all-gather of the build-side columns, so
// that every rank can build the full Index (csvplus.go:707-767) and join its own probe shard against it, plus the
// tiny metadata all-gather that byte-range shards of one file need (quote parity, record counts).
//
// NCCL (NVLink / NVSwitch) is the transport.  The library is bound at run time (dlopen of libnccl.so.2 — the very
// instance torch already mapped when the host is Python) so that single-GPU users need no NCCL at all.
//
// all-gather-v of a table, per column:
//   rank q contributes offsets[0..nrows_q) (uint32, relative to its own data) and its data bytes;
//   every rank receives them at (row base of q, byte base of q) of the concatenated column — one grouped set of
//   ncclSend / ncclRecv (all-gather-v as point-to-point transfers over NVLink) straight into the final buffers: no
//   staging copies, no concat pass;
//   one small kernel then rebases rank q's offsets by (byte base of q - first offset of q).
// Host synchronisations: one (the sizes: rows and bytes per column of every rank).
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <mutex>

#include "core.hpp"
#include "util.cuh"

namespace cpb {

namespace {

struct NcclApi {
    void* lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
};

NcclApi& nccl() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        const char* names[] = {"libnccl.so.2", "libnccl.so", "/usr/lib/x86_64-linux-gnu/libnccl.so.2"};
        for (const char* nm : names) {
            api.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
            if (api.lib) break;
        }
        if (!api.lib) return;
        auto sym = [&](const char* s) { return dlsym(api.lib, s); };
        api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId");
        api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
        api.CommInitAll = (decltype(api.CommInitAll))sym("ncclCommInitAll");
        api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy");
        api.Broadcast = (decltype(api.Broadcast))sym("ncclBroadcast");
        api.AllGather = (decltype(api.AllGather))sym("ncclAllGather");
        api.Send = (decltype(api.Send))sym("ncclSend");
        api.Recv = (decltype(api.Recv))sym("ncclRecv");
        api.GroupStart = (decltype(api.GroupStart))sym("ncclGroupStart");
        api.GroupEnd = (decltype(api.GroupEnd))sym("ncclGroupEnd");
        api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
        if (!api.GetUniqueId || !api.CommInitRank || !api.CommInitAll || !api.CommDestroy || !api.Broadcast || !api.AllGather ||
            !api.GroupStart || !api.GroupEnd || !api.Send || !api.Recv)
            api.lib = nullptr;
    });
    if (!api.lib) throw ArgError{CPB_ERR_UNSUPPORTED, "NCCL (libnccl.so.2) is not available: multi-GPU entry points need it"};
    return api;
}

#define CPB_NCCL(x)                                                                                       \
    do {                                                                                                  \
        ncclResult_t _r = (x);                                                                            \
        if (_r != ncclSuccess) {                                                                          \
            NcclApi& _a = nccl();                                                                         \
            throw ArgError{CPB_ERR_CUDA, std::string("NCCL error in " #x ": ") +                          \
                                             (_a.GetErrorString ? _a.GetErrorString(_r) : "?")};         \
        }                                                                                                 \
    } while (0)

struct Seg { uint64_t row_base, byte_base, rows, first_off; };
constexpr int MAX_RANKS = 64;
struct RebaseParams { int nranks; Seg seg[MAX_RANKS]; uint64_t total_rows, total_bytes; };

// meta per column: (first offset, end offset) of the rows of this view
constexpr int MAX_GATHER_COLS = 128;
struct MetaPtrs { const uint32_t* off[MAX_GATHER_COLS]; };
__global__ void gather_meta_kernel(const __grid_constant__ MetaPtrs mp, int ncols, uint64_t nrows, uint64_t* meta) {
    const int k = threadIdx.x;
    if (k == 0) meta[0] = nrows;
    if (k < ncols) { meta[1 + 2 * k] = mp.off[k][0]; meta[2 + 2 * k] = mp.off[k][nrows]; }
}

}  // namespace

// Pure layout arithmetic of the all-gather-v (also exported for CPU tests): given every rank's (rows, first, end) per
// column, the row / byte base of every rank in the concatenated column.
void allgather_layout(int nranks, int ncols, const uint64_t* meta /* [nranks][1 + 2*ncols] */, uint64_t* row_base /* [nranks+1] */,
                      uint64_t* byte_base /* [ncols][nranks+1] */) {
    const int M = 1 + 2 * ncols;
    row_base[0] = 0;
    for (int q = 0; q < nranks; q++) row_base[q + 1] = row_base[q] + meta[(size_t)q * M];
    for (int k = 0; k < ncols; k++) {
        uint64_t* bb = byte_base + (size_t)k * (nranks + 1);
        bb[0] = 0;
        for (int q = 0; q < nranks; q++) bb[q + 1] = bb[q] + (meta[(size_t)q * M + 2 + 2 * k] - meta[(size_t)q * M + 1 + 2 * k]);
    }
}

namespace {

struct GatherJob {  // one rank's side of a table all-gather
    Ctx* c; const Table* local; int ncols;
    Buf meta_local, meta_all;
    std::vector<uint64_t> meta;  // host copy of meta_all
    std::shared_ptr<Table> out;
};

void job_begin(GatherJob& j) {
    Ctx* c = j.c;
    cudaSetDevice(c->device);
    if (!c->comm) throw ArgError{CPB_ERR_ARG, "this ctx has no communicator (cpb_comm_init_rank / cpb_init_multi)"};
    if (c->nranks > MAX_RANKS) throw ArgError{CPB_ERR_UNSUPPORTED, "more than 64 ranks"};
    j.ncols = (int)j.local->cols.size();
    if (j.ncols > MAX_GATHER_COLS) throw ArgError{CPB_ERR_UNSUPPORTED, "more than 128 columns in an all-gather"};
    const int M = 1 + 2 * j.ncols;
    j.meta_local = dev_alloc(c, M * 8);
    j.meta_all = dev_alloc(c, (size_t)M * 8 * c->nranks);
    MetaPtrs mp{};
    for (int k = 0; k < j.ncols; k++) mp.off[k] = j.local->cols[k].off();
    gather_meta_kernel<<<1, MAX_GATHER_COLS, 0, c->stream>>>(mp, j.ncols, (uint64_t)j.local->nrows, j.meta_local->as<uint64_t>());
    CPB_CUDA(cudaGetLastError());
}
void job_meta_collective(GatherJob& j) {
    Ctx* c = j.c;
    cudaSetDevice(c->device);
    const int M = 1 + 2 * j.ncols;
    CPB_NCCL(nccl().AllGather(j.meta_local->p, j.meta_all->p, (size_t)M, ncclUint64, (ncclComm_t)c->comm, c->stream));
}
void job_sizes(GatherJob& j) {  // the one host round trip
    Ctx* c = j.c;
    cudaSetDevice(c->device);
    const int M = 1 + 2 * j.ncols;
    j.meta = read_back<uint64_t>(c, j.meta_all->p, (size_t)M * c->nranks);
}
void job_data_collective(GatherJob& j) {  // inside ncclGroupStart/End
    Ctx* c = j.c;
    cudaSetDevice(c->device);
    const int R = c->nranks, K = j.ncols, M = 1 + 2 * K;
    std::vector<uint64_t> row_base(R + 1), byte_base((size_t)K * (R + 1));
    allgather_layout(R, K, j.meta.data(), row_base.data(), byte_base.data());
    auto out = std::make_shared<Table>();
    out->ctx = c; out->nrows = (int64_t)row_base[R]; out->first_line = j.local->first_line;
    if (row_base[R] > 0xfffffffeull) throw DataError{CPB_E_TOO_LARGE, -1, 0, false, "gathered table exceeds 2^32-2 rows"};
    for (int k = 0; k < K; k++) {
        const uint64_t* bb = byte_base.data() + (size_t)k * (R + 1);
        if (bb[R] > 0xffffffffull) throw DataError{CPB_E_TOO_LARGE, k, 0, false, "gathered column exceeds 4 GiB"};
        Column col; col.name = j.local->cols[k].name;
        col.offsets = dev_alloc(c, (row_base[R] + 1) * 4);
        col.data = dev_alloc(c, bb[R] + 16);
        // all-gather-v as grouped point-to-point transfers: my segment goes straight to its place in every peer's final
        // buffers over NVLink (a grouped set of ncclBroadcast — one ring per root — was much slower), my own
        // copy is a device-to-device memcpy
        const int me = c->rank;
        const uint64_t my_first = j.meta[(size_t)me * M + 1 + 2 * k];
        const uint64_t my_rows = j.meta[(size_t)me * M], my_bytes = bb[me + 1] - bb[me];
        if (my_rows) CPB_CUDA(cudaMemcpyAsync(col.offsets->as<uint32_t>() + row_base[me], j.local->cols[k].off(), my_rows * 4, cudaMemcpyDeviceToDevice, c->stream));
        if (my_bytes) CPB_CUDA(cudaMemcpyAsync(col.data->as<uint8_t>() + bb[me], j.local->cols[k].bytes() + my_first, my_bytes, cudaMemcpyDeviceToDevice, c->stream));
        for (int q = 0; q < R; q++) {
            if (q == me) continue;
            const uint64_t rows = j.meta[(size_t)q * M], bytes = bb[q + 1] - bb[q];
            if (my_rows) CPB_NCCL(nccl().Send(j.local->cols[k].off(), my_rows, ncclUint32, q, (ncclComm_t)c->comm, c->stream));
            if (my_bytes) CPB_NCCL(nccl().Send(j.local->cols[k].bytes() + my_first, my_bytes, ncclUint8, q, (ncclComm_t)c->comm, c->stream));
            if (rows) CPB_NCCL(nccl().Recv(col.offsets->as<uint32_t>() + row_base[q], rows, ncclUint32, q, (ncclComm_t)c->comm, c->stream));
            if (bytes) CPB_NCCL(nccl().Recv(col.data->as<uint8_t>() + bb[q], bytes, ncclUint8, q, (ncclComm_t)c->comm, c->stream));
        }
        out->cols.push_back(col);
    }
    j.out = out;
}
void job_finish(GatherJob& j) {
    Ctx* c = j.c;
    cudaSetDevice(c->device);
    const int R = c->nranks, K = j.ncols, M = 1 + 2 * K;
    std::vector<uint64_t> row_base(R + 1), byte_base((size_t)K * (R + 1));
    allgather_layout(R, K, j.meta.data(), row_base.data(), byte_base.data());
    uint64_t moved = 0;
    for (int k = 0; k < K; k++) {
        RebaseParams rp{};
        rp.nranks = R; rp.total_rows = row_base[R]; rp.total_bytes = byte_base[(size_t)k * (R + 1) + R];
        for (int q = 0; q < R; q++)
            rp.seg[q] = Seg{row_base[q], byte_base[(size_t)k * (R + 1) + q], j.meta[(size_t)q * M], j.meta[(size_t)q * M + 1 + 2 * k]};
        KernelTimer kt(c, "gather_rebase", (row_base[R] + 1) * 8);
        // off[row_base_q + i] = in_q[i] - first_off_q + byte_base_q ; off[total_rows] = total_bytes
        uint32_t* off = j.out->cols[k].offsets->as<uint32_t>();
        each_row(c, rp.total_rows + 1, [=] __device__(uint64_t i) {
            int q = 0;
            while (q + 1 < rp.nranks && i >= rp.seg[q + 1].row_base) q++;
            off[i] = i == rp.total_rows ? (uint32_t)rp.total_bytes : (uint32_t)((uint64_t)off[i] - rp.seg[q].first_off + rp.seg[q].byte_base);
        });
        moved += rp.total_bytes + rp.total_rows * 4;
    }
    if (c->stats_on) { c->stats["allgather_bytes"].bytes += moved; c->stats["allgather_bytes"].launches += 1; }
}

}  // namespace
}  // namespace cpb

using namespace cpb;

extern "C" {

int cpb_comm_unique_id(uint8_t* id128) {
    return translated(nullptr, nullptr, [&] {
        need(id128, "null id128");
        static_assert(CPB_UNIQUE_ID_BYTES == NCCL_UNIQUE_ID_BYTES, "unique id size");
        ncclUniqueId id;
        CPB_NCCL(nccl().GetUniqueId(&id));
        memcpy(id128, id.internal, NCCL_UNIQUE_ID_BYTES);
        return CPB_OK;
    });
}

int cpb_comm_init_rank(cpb_ctx* h, int nranks, int rank, const uint8_t* id128) {
    return guarded(h, nullptr, [&](Ctx* c) {
        need(id128 && nranks >= 1 && rank >= 0 && rank < nranks, "null id128 or bad rank");
        if (c->comm) throw ArgError{CPB_ERR_ARG, "ctx already has a communicator"};
        ncclUniqueId id;
        memcpy(id.internal, id128, NCCL_UNIQUE_ID_BYTES);
        ncclComm_t comm = nullptr;
        CPB_NCCL(nccl().CommInitRank(&comm, nranks, id, rank));
        c->comm = comm; c->nranks = nranks; c->rank = rank; c->comm_owned = true;
        return CPB_OK;
    });
}

int cpb_init_multi(const int* devices, int n, cpb_ctx** out) {
    if (!devices || !out || n < 1 || n > MAX_RANKS) return CPB_ERR_ARG;
    for (int i = 0; i < n; i++) out[i] = nullptr;
    for (int i = 0; i < n; i++) {
        int st = cpb_init(devices[i], &out[i]);
        if (st != CPB_OK) { for (int j = 0; j < i; j++) { cpb_shutdown(out[j]); out[j] = nullptr; } return st; }
    }
    try {
        std::vector<ncclComm_t> comms(n);
        CPB_NCCL(nccl().CommInitAll(comms.data(), n, devices));
        for (int i = 0; i < n; i++) { Ctx* c = &out[i]->c; c->comm = comms[i]; c->nranks = n; c->rank = i; c->comm_owned = true; }
    } catch (...) {
        int st = translate_exception(&out[0]->c, nullptr);
        for (int i = 0; i < n; i++) { cpb_shutdown(out[i]); out[i] = nullptr; }
        return st;
    }
    return CPB_OK;
}

int cpb_comm_size(cpb_ctx* h) { return h && h->c.comm ? h->c.nranks : 1; }
int cpb_comm_rank(cpb_ctx* h) { return h && h->c.comm ? h->c.rank : 0; }

void cpb_comm_release(cpb::Ctx* c) {  // called by cpb_shutdown
    if (c->comm && c->comm_owned) {
        try { nccl().CommDestroy((ncclComm_t)c->comm); } catch (...) {}
    }
    c->comm = nullptr;
}

// every rank of the communicator calls it (one process per GPU, or one host thread per ctx)
int cpb_allgather_table(cpb_ctx* h, const cpb_table* local, cpb_table** out) {
    return guarded(h, nullptr, [&](Ctx* c) {
        need(local && out, "null local or out");
        *out = nullptr;
        GatherJob j{c, local->t.get()};
        job_begin(j);
        job_meta_collective(j);
        job_sizes(j);
        {
            KernelTimer kt(c, "allgather_nccl", 0, 0);  // device time of the grouped transfers on the ctx stream
            CPB_NCCL(nccl().GroupStart());
            try { job_data_collective(j); } catch (...) { nccl().GroupEnd(); throw; }
            CPB_NCCL(nccl().GroupEnd());
        }
        job_finish(j);
        *out = new cpb_table{j.out};
        return CPB_OK;
    });
}

// single-process form: all n ranks of a cpb_init_multi communicator driven from one host thread (grouped calls)
int cpb_allgather_tables(cpb_ctx* const* hs, const cpb_table* const* locals, int n, cpb_table** outs) {
    if (!hs || !locals || !outs || n < 1) return CPB_ERR_ARG;
    for (int i = 0; i < n; i++) outs[i] = nullptr;
    for (int i = 0; i < n; i++) if (!hs[i] || !locals[i]) return CPB_ERR_ARG;  // before any context is locked
    Ctx* c0 = &hs[0]->c;
    std::vector<std::unique_lock<std::mutex>> locks;  // every rank's context, in rank order
    for (int i = 0; i < n; i++) locks.emplace_back(hs[i]->c.mu);
    return translated(c0, nullptr, [&] {
        if (n != c0->nranks) throw ArgError{CPB_ERR_ARG, "cpb_allgather_tables needs every rank of the communicator"};
        std::vector<GatherJob> jobs;
        for (int i = 0; i < n; i++) jobs.push_back(GatherJob{&hs[i]->c, locals[i]->t.get()});
        for (auto& j : jobs) job_begin(j);
        CPB_NCCL(nccl().GroupStart());
        for (auto& j : jobs) job_meta_collective(j);
        CPB_NCCL(nccl().GroupEnd());
        for (auto& j : jobs) job_sizes(j);
        CPB_NCCL(nccl().GroupStart());
        try { for (auto& j : jobs) job_data_collective(j); } catch (...) { nccl().GroupEnd(); throw; }
        CPB_NCCL(nccl().GroupEnd());
        for (auto& j : jobs) job_finish(j);
        for (int i = 0; i < n; i++) outs[i] = new cpb_table{jobs[i].out};
        return CPB_OK;
    });
}

// small metadata exchange (host values in, host values out): quote parity / record counts of byte-range shards
int cpb_allgather_u64(cpb_ctx* h, const uint64_t* in, int count, uint64_t* out) {
    return guarded(h, nullptr, [&](Ctx* c) {
        need(in && out && count >= 1, "null in or out, or no values");
        if (!c->comm) { memcpy(out, in, (size_t)count * 8); return CPB_OK; }
        Buf a = dev_alloc(c, (size_t)count * 8), b = dev_alloc(c, (size_t)count * 8 * c->nranks);
        uint64_t* hp = (uint64_t*)c->pinned_scratch((size_t)count * 8 * (c->nranks + 1));
        memcpy(hp, in, (size_t)count * 8);
        CPB_CUDA(cudaMemcpyAsync(a->p, hp, (size_t)count * 8, cudaMemcpyHostToDevice, c->stream));
        CPB_NCCL(nccl().AllGather(a->p, b->p, (size_t)count, ncclUint64, (ncclComm_t)c->comm, c->stream));
        CPB_CUDA(cudaMemcpyAsync(hp + count, b->p, (size_t)count * 8 * c->nranks, cudaMemcpyDeviceToHost, c->stream));
        sync_stream(c);
        memcpy(out, hp + count, (size_t)count * 8 * c->nranks);
        return CPB_OK;
    });
}

// the layout arithmetic alone (pure host code; CPU tests call it without a GPU)
int cpb_allgather_layout(int nranks, int ncols, const uint64_t* meta, uint64_t* row_base, uint64_t* byte_base) {
    if (nranks < 1 || ncols < 0 || !meta || !row_base || (ncols && !byte_base)) return CPB_ERR_ARG;
    allgather_layout(nranks, ncols, meta, row_base, byte_base);
    return CPB_OK;
}

}  // extern "C"
