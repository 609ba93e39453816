// stream.cu — inputs of any size, parsed in batches of whole records (cpb_stream_*; DESIGN.md §3.7).
//
// Replaces (reference): the record-at-a-time pull of Reader.Iterate (csvplus.go:1080-1146), whose memory does not grow
// with the input.  Here the input arrives in host pushes; each batch is cut at the end of its last complete record ON
// THE GPU, parsed as a self-contained CSV input, and the tail is carried to the front of the next batch.
//
// The cut.  A batch starts at a record start, so the quote state there is "outside".
//   * default options, TrimLeadingSpace: in valid input every '"' is structural or half of an escaped pair, so the
//     parity of the quotes before a '\n' decides whether it ends a line.  stream_cut_kernel reads the batch once with
//     aligned 16-byte loads: each CTA summarises a 64 KiB chunk (quote parity; for entry parity 0 and 1 the last '\n'
//     outside quotes), the last CTA to finish (atomic ticket) prefix-XORs the parities and takes the last chunk that
//     has a qualifying newline.
//   * CommentChar / LazyQuotes: a quote in a comment line or a lazy bare quote breaks parity; the record-boundary DFA of
//     parse_general.cu decides instead (general_cut).
// Malformed input only ever moves the cut later than the first error (parity counts a bare quote; an unclosed quote
// keeps every later newline "inside"), so the failing record is parsed whole and the first error and its line are the
// whole-input parse's.  An unclosed quote running to EOF makes the carried tail grow to the end of the input.
#include <algorithm>

#include "core.hpp"
#include "util.cuh"

namespace cpb {

void general_cut(Ctx* c, const uint8_t* in, uint64_t n, const cpb_reader_opts& o, uint64_t* cut_dev);  // parse_general.cu

namespace {

constexpr uint32_t CUT_CHUNK = 64u << 10;  // bytes per CTA
constexpr int CUT_THREADS = 256;           // 8 warps x 8 KiB, 16 rounds of 512 contiguous bytes per warp
constexpr uint32_t WARP_BYTES = CUT_CHUNK / (CUT_THREADS / 32);

__device__ __forceinline__ uint32_t prefix_xor16(uint32_t m) {  // bit i = XOR of bits 0..i
    m ^= m << 1; m ^= m << 2; m ^= m << 4; m ^= m << 8;
    return m & 0xffffu;
}

// summ[chunk] = {quote parity, cut if entered outside quotes, cut if entered inside, 0}: cuts are chunk offsets + 1 of a
// '\n', 0 = none.  *out = the cut of [0, n) (0: no complete record).  ticket and *out start at 0.
__global__ void __launch_bounds__(CUT_THREADS) stream_cut_kernel(const uint8_t* __restrict__ in, uint64_t n, uint4* summ,
                                                                  uint32_t* ticket, unsigned long long* out) {
    __shared__ uint32_t wpar[CUT_THREADS / 32], wl[2][CUT_THREADS / 32];
    __shared__ uint32_t last_cta;
    __shared__ unsigned long long best_of[CUT_THREADS / 32];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t cbase = (uint64_t)blockIdx.x * CUT_CHUNK;
    uint32_t wq = 0, l0 = 0, l1 = 0;  // parity of the warp's bytes so far; last newline at warp-relative parity 0 / 1
    for (int r = 0; r < (int)(WARP_BYTES / 512); r++) {
        const uint32_t off = warp * WARP_BYTES + (uint32_t)r * 512 + lane * 16;
        const uint64_t p = cbase + off;
        uint32_t qm = 0, nm = 0;
        if (p + 16 <= n) {
            const uint4 x = *reinterpret_cast<const uint4*>(in + p);
            qm = flags16(eq_flags(x.x, 0x22222222u), eq_flags(x.y, 0x22222222u), eq_flags(x.z, 0x22222222u), eq_flags(x.w, 0x22222222u));
            nm = flags16(eq_flags(x.x, 0x0a0a0a0au), eq_flags(x.y, 0x0a0a0a0au), eq_flags(x.z, 0x0a0a0a0au), eq_flags(x.w, 0x0a0a0a0au));
        } else if (p < n) {
            for (uint32_t j = 0; j < (uint32_t)(n - p); j++) { qm |= (uint32_t)(in[p + j] == '"') << j; nm |= (uint32_t)(in[p + j] == '\n') << j; }
        }
        const uint32_t mine = __popc(qm) & 1u;
        uint32_t inc = mine;  // inclusive XOR scan over the lanes
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= (uint32_t)d) inc ^= t;
        }
        uint32_t inside = prefix_xor16(qm);  // a '\n' is no quote: inclusive parity at it = parity before it
        if (wq ^ inc ^ mine) inside ^= 0xffffu;
        const uint32_t o0 = nm & ~inside, o1 = nm & inside;
        if (o0) l0 = off + 32 - __clz(o0);
        if (o1) l1 = off + 32 - __clz(o1);
        wq ^= __shfl_sync(0xffffffffu, inc, 31);
    }
    l0 = __reduce_max_sync(0xffffffffu, l0);
    l1 = __reduce_max_sync(0xffffffffu, l1);
    if (lane == 0) { wpar[warp] = wq; wl[0][warp] = l0; wl[1][warp] = l1; }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t par = 0, c0 = 0, c1 = 0;
        for (int w = 0; w < CUT_THREADS / 32; w++) {
            if (wl[par][w]) c0 = wl[par][w];
            if (wl[par ^ 1][w]) c1 = wl[par ^ 1][w];
            par ^= wpar[w];
        }
        summ[blockIdx.x] = make_uint4(par, c0, c1, 0);
        __threadfence();
        last_cta = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last_cta) return;
    __threadfence();
    // ---- the last CTA: chunk entry parities (prefix XOR) and the last chunk with a qualifying newline
    const uint32_t nch = gridDim.x, per = (nch + CUT_THREADS - 1) / CUT_THREADS;
    const uint32_t lo = min(nch, threadIdx.x * per), hi = min(nch, lo + per);
    uint32_t mine = 0;
    for (uint32_t k = lo; k < hi; k++) mine ^= __ldcg(&summ[k].x);
    uint32_t inc = mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= (uint32_t)d) inc ^= t;
    }
    if (lane == 31) wpar[warp] = inc;
    __syncthreads();
    uint32_t e = inc ^ mine;
    for (uint32_t w = 0; w < warp; w++) e ^= wpar[w];
    unsigned long long best = 0;
    for (uint32_t k = lo; k < hi; k++) {
        const uint4 s = __ldcg(&summ[k]);
        const uint32_t cut = e ? s.z : s.y;
        if (cut) best = (unsigned long long)k * CUT_CHUNK + cut;
        e ^= s.x;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, d));
    if (lane == 0) best_of[warp] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 0; w < CUT_THREADS / 32; w++) best = max(best, best_of[w]);
        *out = best;
    }
}

}  // namespace

// enqueues the cut of [0, n) into *cut_dev (8 bytes of device memory) on the ctx stream
void stream_cut(Ctx* c, const uint8_t* in, uint64_t n, const cpb_reader_opts& o, uint64_t* cut_dev) {
    if (o.comment != 0 || o.lazy_quotes) { general_cut(c, in, n, o, cut_dev); return; }
    CPB_CUDA(cudaMemsetAsync(cut_dev, 0, 16, c->stream));  // the cut and the ticket behind it
    if (n == 0) return;
    const uint64_t nch = (n + CUT_CHUNK - 1) / CUT_CHUNK;
    if (nch > 0x7fffffffull) throw ArgError{CPB_ERR_ARG, "stream batch too large"};
    Buf summ = dev_alloc(c, nch * 16);
    KernelTimer kt(c, "stream_cut", n);
    stream_cut_kernel<<<(uint32_t)nch, CUT_THREADS, 0, c->stream>>>(in, n, summ->as<uint4>(), reinterpret_cast<uint32_t*>(cut_dev + 1),
                                                                    reinterpret_cast<unsigned long long*>(cut_dev));
    CPB_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------ the stream object
// Two device staging slots.  The current slot holds [carried tail | pushed bytes]; once a batch is cut, its tail is
// copied device-to-device to the front of the other slot and the next pushes land behind it, so every batch starts
// 16-byte aligned.  Host->device copies run on the stream's own copy stream, which waits for the event recorded after
// the last parse (and tail copy) that read the slot: the copy of batch b+1 overlaps what the caller does with batch b.
struct Stream {
    Ctx* c;
    cpb_reader_opts o;
    std::vector<std::pair<std::string, int>> spec;
    const cpb_pred* filter;
    cudaStream_t copy = nullptr;
    cudaEvent_t copied = nullptr;   // after the last push's copy (the parse waits for it)
    cudaEvent_t freed[2] = {};      // after the last ctx-stream work that read slot k
    Buf slot[2];
    uint64_t cap[2] = {0, 0};
    int cur = 0;
    uint64_t len = 0;               // bytes in the current slot
    bool last_pushed = false, done = false, resolved = false;
    uint64_t line_base = 0;         // DataSourceError.Line of the next batch's first data record
    uint64_t max_push = 0;          // largest push so far
    uint64_t trial_at = 0;          // carried bytes without a cut at which the tail is trial-parsed (see next())
    Buf cut_dev;

    ~Stream() {
        if (copy) cudaStreamSynchronize(copy);
        cudaStreamSynchronize(c->stream);
        slot[0].reset(); slot[1].reset(); cut_dev.reset();
        if (copied) cudaEventDestroy(copied);
        for (auto e : freed) if (e) cudaEventDestroy(e);
        if (copy) cudaStreamDestroy(copy);
    }

    static uint64_t slot_class(uint64_t b) {  // 32 MiB steps: slots of similar batches are served by the same pool blocks
        return (b + 256 + (32u << 20) - 1) / (32u << 20) * (32u << 20);
    }
    // slot k holds at least `need` bytes (+ zero padding), keeping its first `keep` bytes; ctx-stream ordered
    void reserve(int k, uint64_t need, uint64_t keep) {
        if (need + 256 <= cap[k]) return;
        const uint64_t nc = slot_class(need);
        Buf nb = dev_alloc(c, nc);
        if (keep) CPB_CUDA(cudaStreamWaitEvent(c->stream, copied, 0));  // pushes still landing in the old block
        if (keep) CPB_CUDA(cudaMemcpyAsync(nb->p, slot[k]->p, keep, cudaMemcpyDeviceToDevice, c->stream));
        slot[k] = nb; cap[k] = nc;
        CPB_CUDA(cudaEventRecord(freed[k], c->stream));  // the copy stream must see the new block and the kept bytes
    }

    void push(const void* bytes, uint64_t n, bool is_last) {
        if (done || last_pushed) throw ArgError{CPB_ERR_ARG, "cpb_stream_push after the last push"};
        reserve(cur, len + n, len);
        if (n) {
            CPB_CUDA(cudaStreamWaitEvent(copy, freed[cur], 0));
            CPB_CUDA(cudaMemcpyAsync(slot[cur]->as<uint8_t>() + len, bytes, n, cudaMemcpyHostToDevice, copy));
            CPB_CUDA(cudaEventRecord(copied, copy));
        }
        len += n;
        last_pushed = is_last;
        max_push = std::max(max_push, n);
    }

    // -> the next batch (table null: no complete record yet)
    Parsed next() {
        bool trial = false;
        if (done || (!last_pushed && len == 0)) return {};  // (nothing pushed yet: no slot either)
        CPB_CUDA(cudaStreamWaitEvent(c->stream, copied, 0));
        uint8_t* in = slot[cur]->as<uint8_t>();
        CPB_CUDA(cudaMemsetAsync(in + len, 0, std::min<uint64_t>(cap[cur] - len, 256), c->stream));
        uint64_t cut = len;
        if (!last_pushed) {
            stream_cut(c, in, len, o, cut_dev->as<uint64_t>());
            cut = read_back<uint64_t>(c, cut_dev->p);
            if (cut == 0) {
                // No line end outside quotes.  Either one record is longer than what was pushed so far, or (default
                // options) a bare quote flipped the quote parity for the rest of the input, and the reference would stop
                // at that record.  As the tail grows (at 4, 8, 16, ... times the largest push), it is parsed as if it
                // ended the input: an error that the missing rest cannot have caused ends the stream there.
                if (len < std::max(trial_at, 4 * max_push)) return {};
                trial_at = 2 * len;
                cut = len;
                trial = true;
            } else trial_at = 0;
        }
        // until the first record has been seen, a batch is parsed as the start of the input (header, field count);
        // afterwards with the resolved (name, field) pairs, no header row and the first record's field count
        cpb_reader_opts bo = o;
        if (resolved) bo.header_from_first_row = 0;
        const uint64_t base = resolved ? line_base : (o.header_from_first_row ? 2u : 1u);
        Parsed p = parse_csv(c, in, cut, bo, spec, filter, base);
        if (trial) {
            // a bare quote is an error wherever the record ends; another error only if a later record starts after it
            const bool sure = p.error && p.error->has_line && (p.error->kind == CPB_E_BARE_QUOTE || p.error->line + 1 < base + p.records);
            if (!sure) return {};
        }
        if (!resolved) {
            if (p.no_record && !last_pushed) {
                p.error.reset();  // only blank / comment lines so far: they hold no record, drop them
                p.table = nullptr;
            } else if (!p.error) {
                resolved = true;
                const Table& t = *p.table;
                if (o.header_from_first_row) {
                    spec.clear();
                    for (size_t i = 0; i < t.cols.size(); i++) spec.emplace_back(t.cols[i].name, t.src_field[i]);
                }
                if (o.num_fields == 0) o.num_fields = t.record_fields;
                line_base = (o.header_from_first_row ? 2 : 1) + p.records;
            }
        } else line_base += p.records;
        if (p.error || last_pushed) {
            // the input is parsed (the tables own their bytes): the slots go back to the pool now, stream-ordered after
            // the parse, instead of staying allocated through the caller's plan until the stream is freed
            done = true;
            slot[0].reset(); slot[1].reset();
            cap[0] = cap[1] = 0;
            return p;
        }
        // carry [cut, len) to the front of the other slot
        const int nx = cur ^ 1;
        const uint64_t tail = len - cut;
        reserve(nx, tail, 0);
        if (tail) CPB_CUDA(cudaMemcpyAsync(slot[nx]->p, in + cut, tail, cudaMemcpyDeviceToDevice, c->stream));
        CPB_CUDA(cudaEventRecord(freed[cur], c->stream));
        CPB_CUDA(cudaEventRecord(freed[nx], c->stream));
        cur = nx; len = tail;
        return p;
    }
};

Stream* stream_open(Ctx* c, const cpb_reader_opts& o, std::vector<std::pair<std::string, int>> spec, const cpb_pred* filter) {
    // invalid options are reported by the first batch's parse, as cpb_parse_csv reports them
    auto s = new Stream{c, o, std::move(spec), filter};
    try {
        CPB_CUDA(cudaStreamCreateWithFlags(&s->copy, cudaStreamNonBlocking));
        CPB_CUDA(cudaEventCreateWithFlags(&s->copied, cudaEventDisableTiming));
        for (auto& e : s->freed) CPB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        for (auto& e : s->freed) CPB_CUDA(cudaEventRecord(e, c->stream));
        CPB_CUDA(cudaEventRecord(s->copied, s->copy));
        s->cut_dev = dev_alloc(c, 16);  // the first slot is allocated by the first push, at that push's size
    } catch (...) {
        delete s;
        throw;
    }
    return s;
}
void stream_push(Stream* s, const void* bytes, uint64_t n, bool is_last) { s->push(bytes, n, is_last); }
Parsed stream_next(Stream* s, bool* done) {
    Parsed p = s->next();
    *done = s->done;
    return p;
}
void stream_free(Stream* s) { delete s; }
Ctx* stream_ctx(Stream* s) { return s->c; }

}  // namespace cpb
