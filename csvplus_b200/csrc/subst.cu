// subst.cu — multi-byte runes of the Reader options (csvplus.go:971-993): a Delimiter / CommentChar >= U+0080 and the
// multi-byte Unicode spaces TrimLeadingSpace trims (encoding/csv trims with unicode.IsSpace: U+0085, U+00A0, U+1680,
// U+2000-U+200A, U+2028, U+2029, U+202F, U+205F, U+3000).
//
// The scan kernels and the record-boundary DFA work on single bytes.  Instead of widening them, the input is
// transcoded once: every occurrence of such a rune's UTF-8 sequence is replaced by ONE byte value that does not occur
// anywhere in the input (found with a 256-bin histogram).  UTF-8 lead bytes never equal continuation bytes, so the
// occurrences of distinct encoded runes cannot overlap and "leftmost byte-sequence match" — what bytes.IndexRune /
// utf8.DecodeRune give the reference — is simply "every occurrence".  The kernels then see a single-byte delimiter /
// comment / space class; wherever such a byte is DATA (inside a quoted field, or a space that is not leading) the
// sequential record machine's sink expands it back to the original sequence (SubTable), so values stay bit-exact.
// Errors are reported by record ordinal, never by byte position, so shifting positions changes nothing visible.
#include <algorithm>

#include "core.hpp"
#include "util.cuh"
#include "subst.hpp"

namespace cpb {

namespace {

constexpr int SUB_CHUNK = 512;
struct SeqDev { int n; uint8_t len[MAX_SUB_SEQ]; uint8_t b[MAX_SUB_SEQ][4]; uint8_t sub[MAX_SUB_SEQ]; };

__global__ void hist256_kernel(const uint8_t* __restrict__ in, uint64_t n, unsigned long long* hist) {
    __shared__ uint32_t sh[256];
    sh[threadIdx.x] = 0;
    __syncthreads();
    for (uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * 16; i < n; i += (uint64_t)gridDim.x * blockDim.x * 16) {
        if (i + 16 <= n) {
            const uint4 v = *reinterpret_cast<const uint4*>(in + i);
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int j = 0; j < 4; j++) {
                atomicAdd(&sh[w[j] & 255u], 1u); atomicAdd(&sh[(w[j] >> 8) & 255u], 1u);
                atomicAdd(&sh[(w[j] >> 16) & 255u], 1u); atomicAdd(&sh[w[j] >> 24], 1u);
            }
        } else for (uint64_t k = i; k < n; k++) atomicAdd(&sh[in[k]], 1u);
    }
    __syncthreads();
    if (sh[threadIdx.x]) atomicAdd(&hist[threadIdx.x], (unsigned long long)sh[threadIdx.x]);
}

// the sequence starting at i, if any: its index or -1
__device__ __forceinline__ int match_at(const uint8_t* __restrict__ in, uint64_t n, uint64_t i, const SeqDev& sd) {
    const uint8_t b0 = in[i];
    if (b0 < 0x80) return -1;
    for (int q = 0; q < sd.n; q++) {
        if (sd.b[q][0] != b0 || i + sd.len[q] > n) continue;
        bool ok = true;
        for (int j = 1; j < sd.len[q]; j++) ok = ok && in[i + j] == sd.b[q][j];
        if (ok) return q;
    }
    return -1;
}
// one thread per 512-byte chunk (the rare path: simplicity over bandwidth); WRITE: transcode, else count output bytes
template <bool WRITE>
__global__ void subst_kernel(const uint8_t* __restrict__ in, uint64_t n, SeqDev sd, uint32_t* counts, const uint32_t* __restrict__ offs, uint8_t* out) {
    const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t lo = c * SUB_CHUNK;
    if (lo >= n) return;
    const uint64_t hi = lo + SUB_CHUNK < n ? lo + SUB_CHUNK : n;
    uint64_t i = lo;
    for (uint64_t back = 1; back <= 3 && back <= lo; back++) {  // a match that started before the chunk covers its first bytes
        const int q = match_at(in, n, lo - back, sd);
        if (q >= 0 && sd.len[q] > back) i = lo - back + sd.len[q];
    }
    uint32_t k = 0;
    uint8_t* o = WRITE ? out + offs[c] : nullptr;
    while (i < hi) {
        const int q = match_at(in, n, i, sd);
        if (q >= 0) { if (WRITE) o[k] = sd.sub[q]; k++; i += sd.len[q]; }
        else { if (WRITE) o[k] = in[i]; k++; i++; }
    }
    if (!WRITE) counts[c] = k;
}

}  // namespace

std::string utf8_rune(uint32_t r) {
    std::string s;
    if (r < 0x80) s += (char)r;
    else if (r < 0x800) { s += (char)(0xC0 | (r >> 6)); s += (char)(0x80 | (r & 0x3F)); }
    else if (r < 0x10000) { s += (char)(0xE0 | (r >> 12)); s += (char)(0x80 | ((r >> 6) & 0x3F)); s += (char)(0x80 | (r & 0x3F)); }
    else { s += (char)(0xF0 | (r >> 18)); s += (char)(0x80 | ((r >> 12) & 0x3F)); s += (char)(0x80 | ((r >> 6) & 0x3F)); s += (char)(0x80 | (r & 0x3F)); }
    return s;
}

bool needs_substitution(const cpb_reader_opts& o) { return o.delimiter >= 0x80 || o.comment >= 0x80 || o.trim_leading_space; }

// Transcodes `in` when the options name multi-byte runes that occur in it.  Returns the buffer to parse (null: parse
// `in` as it is), the single-byte delimiter / comment to use and the expansion table.
Substitution substitute_runes(Ctx* c, const uint8_t* in, uint64_t n, const cpb_reader_opts& o) {
    Substitution r;
    r.delimiter = o.delimiter; r.comment = o.comment;
    struct Want { std::string seq; int kind; };  // kind 0 delimiter, 1 comment, 2 space
    std::vector<Want> want;
    if (o.delimiter >= 0x80) want.push_back({utf8_rune(o.delimiter), 0});
    if (o.comment >= 0x80) want.push_back({utf8_rune(o.comment), 1});
    if (o.trim_leading_space)
        for (uint32_t s : kUnicodeSpaces) if (s != o.delimiter && s != o.comment) want.push_back({utf8_rune(s), 2});
    if (want.empty()) return r;
    // ---- which byte values occur
    Buf hist = dev_alloc(c, 256 * 8);
    CPB_CUDA(cudaMemsetAsync(hist->p, 0, 256 * 8, c->stream));
    if (n) {
        KernelTimer kt(c, "subst_hist", n);
        hist256_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(in, n, (unsigned long long*)hist->p);
        CPB_CUDA(cudaGetLastError());
    }
    const std::vector<unsigned long long> hh = read_back<unsigned long long>(c, hist->p, 256);
    std::vector<int> unused;
    auto reserved = [&](int b) {
        return b == 0 || b == '"' || b == '\n' || b == '\r' || b == ' ' || b == '\t' || b == '\v' || b == '\f' || (uint32_t)b == o.delimiter ||
               (uint32_t)b == o.comment;
    };
    for (int b = 1; b < 0x80; b++) if (hh[b] == 0 && !reserved(b)) unused.push_back(b);
    SeqDev sd{};
    SubTable tab{};
    size_t next_unused = 0;
    for (auto& w : want) {
        bool occurs = true;
        for (unsigned char ch : w.seq) occurs = occurs && hh[ch] != 0;
        if (!occurs && w.kind == 2) continue;  // a space that cannot occur needs nothing
        if (next_unused >= unused.size())
            throw ArgError{CPB_ERR_UNSUPPORTED, "multi-byte reader runes: the input uses every ASCII byte value, none is free to stand in"};
        const uint8_t sub = (uint8_t)unused[next_unused++];
        if (w.kind == 0) r.delimiter = sub;
        else if (w.kind == 1) r.comment = sub;
        else tab.space_bits[sub >> 5] |= 1u << (sub & 31);
        tab.bits[sub >> 5] |= 1u << (sub & 31);
        tab.len[sub] = (uint8_t)w.seq.size();
        for (size_t j = 0; j < w.seq.size(); j++) tab.seq[sub][j] = (uint8_t)w.seq[j];
        if (occurs) {
            sd.len[sd.n] = (uint8_t)w.seq.size();
            for (size_t j = 0; j < w.seq.size(); j++) sd.b[sd.n][j] = (uint8_t)w.seq[j];
            sd.sub[sd.n] = sub;
            sd.n++;
        }
    }
    r.table = dev_alloc(c, sizeof(SubTable));
    {
        SubTable* ht = (SubTable*)c->pinned_scratch(sizeof(SubTable));
        *ht = tab;
        CPB_CUDA(cudaMemcpyAsync(r.table->p, ht, sizeof(SubTable), cudaMemcpyHostToDevice, c->stream));
        sync_stream(c);  // the pinned scratch is reused below
    }
    r.host_table = tab;
    if (sd.n == 0 || n == 0) return r;  // nothing to transcode: the stand-in bytes simply never occur
    if (n > 0xfff00000ull) throw ArgError{CPB_ERR_UNSUPPORTED, "multi-byte reader runes: inputs of 4 GiB and more must be parsed in batches"};
    // ---- count, scan, transcode
    const uint64_t nchunks = (n + SUB_CHUNK - 1) / SUB_CHUNK;
    Buf counts = dev_alloc(c, (nchunks + 1) * 4), tot = dev_alloc(c, 8);
    {
        KernelTimer kt(c, "subst_count", n);
        subst_kernel<false><<<(uint32_t)((nchunks + 127) / 128), 128, 0, c->stream>>>(in, n, sd, counts->as<uint32_t>(), nullptr, nullptr);
        CPB_CUDA(cudaGetLastError());
    }
    exclusive_scan_u32(c, counts->as<uint32_t>(), counts->as<uint32_t>(), nchunks, tot->as<uint64_t>());
    r.nbytes = read_back<uint64_t>(c, tot->p);
    r.buffer = dev_alloc(c, ((r.nbytes + 15) & ~15ull) + 256);
    CPB_CUDA(cudaMemsetAsync(r.buffer->as<uint8_t>() + (r.nbytes & ~15ull), 0, ((r.nbytes + 15) & ~15ull) + 256 - (r.nbytes & ~15ull), c->stream));
    {
        KernelTimer kt(c, "subst_write", n + r.nbytes);
        subst_kernel<true><<<(uint32_t)((nchunks + 127) / 128), 128, 0, c->stream>>>(in, n, sd, nullptr, counts->as<uint32_t>(), r.buffer->as<uint8_t>());
        CPB_CUDA(cudaGetLastError());
    }
    return r;
}

}  // namespace cpb
