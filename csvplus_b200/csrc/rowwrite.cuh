// rowwrite.cuh — how rows become bytes, for every row serialiser: ToCsv (write.cu), ToJSON (json.cu), Index.WriteTo
// (gob.cu), Sprintf / ToText (sprintf.cu) and FormatInt / FormatFloat (format.cu).
//
// Each serialiser is a row type R, a trivially copyable struct passed to the kernels by value (as a __grid_constant__
// parameter, so its pointer arrays stay in parameter space however they are indexed):
//   __device__ uint64_t len(uint64_t r) const           the output bytes of row r (not needed by FormatInt / FormatFloat,
//                                                        whose digit kernels write the lengths)
//   R::Tables, TABLE_BYTES                               what write reads from shared memory, at most TABLE_BYTES bytes
//   uint32_t tail() const, TAIL_VARIES                   (host) the bytes of them this launch copies, <= TABLE_BYTES;
//                                                        whether that differs from launch to launch
//   __device__ Tables stage(uint8_t* sm) const           copies them to sm and says where they are (a block-wide step)
//   __device__ void write(uint64_t r, uint8_t* q, const Tables&) const    writes row r at q
// A row type without tables derives from NoTables.
//
// A sink then runs: row_lengths (one thread per row, saturated at 0xFFFFFFFF) -> row_offsets (exclusive_scan_u32, one
// readback of the exact total, check_body) -> its room check and allocation -> row_write (warp_write_rows).
#pragma once
#include <algorithm>

#include "core.hpp"
#include "util.cuh"

namespace cpb {

// Go's utf8.DecodeRune: the length of the valid UTF-8 sequence starting at p (rem >= 1 bytes readable), 0 if none
__host__ __device__ __forceinline__ uint32_t utf8_seq(const uint8_t* p, uint64_t rem) {
    const uint8_t c = p[0];
    if (c < 0xC2) return 0;  // ASCII, a continuation byte, or an overlong lead C0 / C1
    if (c <= 0xDF) return rem >= 2 && (p[1] & 0xC0) == 0x80 ? 2 : 0;
    if (c <= 0xEF) {
        const uint8_t lo = c == 0xE0 ? 0xA0 : 0x80, hi = c == 0xED ? 0x9F : 0xBF;
        return rem >= 3 && p[1] >= lo && p[1] <= hi && (p[2] & 0xC0) == 0x80 ? 3 : 0;
    }
    if (c <= 0xF4) {
        const uint8_t lo = c == 0xF0 ? 0x90 : 0x80, hi = c == 0xF4 ? 0x8F : 0xBF;
        return rem >= 4 && p[1] >= lo && p[1] <= hi && (p[2] & 0xC0) == 0x80 && (p[3] & 0xC0) == 0x80 ? 4 : 0;
    }
    return 0;
}

// One warp serialises 32 consecutive rows.  Their output bytes are contiguous, so every lane writes its row into the
// warp's shared-memory stage, laid out like the destination, and the warp stores the stage with aligned 16-byte vectors
// (a thread-per-row kernel storing bytes straight to HBM touches ~20 sectors per store instruction).  A group longer
// than the stage (very long rows) is written directly.
//   stages  the block's WARPS stages of STAGE + 16 bytes each, 16-byte aligned
//   pos     the n + 1 output offsets of the rows
//   row     row(r, q) serialises row r starting at q (in the stage or in out)
template <int WARPS, uint32_t STAGE, class Row>
__device__ __forceinline__ void warp_write_rows(uint8_t* stages, uint64_t n, const uint32_t* __restrict__ pos, uint8_t* out, Row row) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint8_t* stage = stages + warp * (int)(STAGE + 16);  // signed: with an unsigned offset ptxas spills in the JSON writer
    const uint64_t nwarps = (uint64_t)gridDim.x * WARPS;
    for (uint64_t g = (uint64_t)blockIdx.x * WARPS + warp; g * 32 < n; g += nwarps) {
        const uint64_t r = g * 32 + lane;
        const bool valid = r < n;
        const uint32_t d = valid ? pos[r] : 0u;
        const uint64_t lastr = g * 32 + 31 < n ? g * 32 + 31 : n - 1;
        const uint32_t d0 = __shfl_sync(0xffffffffu, d, 0), dend = pos[lastr + 1];
        // the absolute destination is out + d; alignment is that of the pointer, not of the offset alone
        const uint32_t sh = (uint32_t)((reinterpret_cast<uintptr_t>(out) + d0) & 15u), total = dend - d0;
        const bool staged = (uint64_t)sh + total <= STAGE;  // 64-bit: a group of 4 GiB - 15 bytes or more must not wrap
        if (valid) row(r, staged ? stage + sh + (d - d0) : out + d);
        if (staged) {
            __syncwarp();
            uint8_t* gb = out + d0 - sh;
            for (uint32_t x = lane * 16; x < sh + total; x += 32 * 16) {
                if (x >= sh && x + 16 <= sh + total) *reinterpret_cast<uint4*>(gb + x) = *reinterpret_cast<const uint4*>(stage + x);
                else for (uint32_t y = x; y < x + 16; y++) if (y >= sh && y < sh + total) gb[y] = stage[y];
            }
            __syncwarp();
        }
    }
}

struct NoTables {
    struct Tables {};
    static constexpr uint32_t TABLE_BYTES = 0;
    static constexpr bool TAIL_VARIES = false;
    uint32_t tail() const { return 0; }
    __device__ Tables stage(uint8_t*) const { return {}; }
};

// len[r] = the bytes of row r, saturated at 0xFFFFFFFF (a saturated total is then refused by check_body); with SUM,
// *sum += the exact 64-bit total of the rows
template <class R, bool SUM>
__global__ void row_len_kernel(const __grid_constant__ R rows, uint64_t n, uint32_t* __restrict__ len, unsigned long long* sum) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t total = 0;
    if (r < n) {
        total = rows.len(r);
        len[r] = total > 0xffffffffull ? 0xffffffffu : (uint32_t)total;
    }
    if constexpr (SUM) {
        total = warp_sum_u64(total);
        if ((threadIdx.x & 31) == 0 && total) atomicAdd(sum, (unsigned long long)total);
    }
}

constexpr int ROW_WARPS = 8;  // warps per block of row_write_kernel
// The blocks of row_write_kernel an SM holds (228 KB of shared memory per SM on sm_90, 1 KB of it reserved per block),
// given to ptxas, which cannot see dynamic shared memory, so that it spends the registers that residency leaves; 0 (no
// bound) when the tables' size varies from launch to launch.
template <class R, uint32_t STAGE>
constexpr uint32_t row_blocks() {
    const uint32_t smem = ROW_WARPS * (STAGE + 16) + R::TABLE_BYTES + 1024;
    return R::TAIL_VARIES ? 0 : std::min<uint32_t>(2048 / (ROW_WARPS * 32), (228u << 10) / smem);
}

// dynamic shared memory: the ROW_WARPS stages of STAGE + 16 bytes, then the row type's tables
template <class R, uint32_t STAGE>
__global__ void __launch_bounds__(ROW_WARPS * 32, (row_blocks<R, STAGE>()))
    row_write_kernel(const __grid_constant__ R rows, uint64_t n, const uint32_t* __restrict__ pos, uint8_t* out) {
    extern __shared__ __align__(16) uint8_t smem[];
    const typename R::Tables tables = rows.stage(smem + ROW_WARPS * (STAGE + 16));
    warp_write_rows<ROW_WARPS, STAGE>(smem, n, pos, out, [&](uint64_t r, uint8_t* q) { rows.write(r, q, tables); });
}

// the lengths of rows [0, n) into len, timed as `timer` with `bytes` algorithmic bytes; with SUM, *sum (zeroed by the
// caller) += their exact total
template <bool SUM = false, class R>
void row_lengths(Ctx* c, const R& rows, uint64_t n, uint32_t* len, const char* timer, uint64_t bytes, unsigned long long* sum = nullptr) {
    if (!n) return;
    KernelTimer kt(c, timer, bytes);
    row_len_kernel<R, SUM><<<nblk(n, 256), 256, 0, c->stream>>>(rows, n, len, sum);
    CPB_CUDA(cudaGetLastError());
}

// Offsets are 32-bit, so a body of 4 GiB or more is refused (CPB_E_TOO_LARGE, what): above max_body (MAX_BODY for
// ToCsv and Sprintf; MAX_BODY - 1 for ToJSON, whose closing ']' follows the body, and WriteTo), and as one row of
// exactly MAX_BODY bytes, which may be a saturated longer one
constexpr uint64_t MAX_BODY = 0xffffffffull;
inline void check_body(uint64_t body, uint64_t n, uint64_t max_body, const std::string& what) {
    if (body > max_body || (n == 1 && body == MAX_BODY)) throw DataError{CPB_E_TOO_LARGE, -1, 0, false, what};
}

// the lengths at len (n + 1 entries) become the offsets; one readback of tot[0, words): the exact total of the lengths,
// then the words - 1 values the caller's earlier launches left after it; the total is checked by check_body
inline std::vector<uint64_t> row_offsets(Ctx* c, uint32_t* len, uint64_t n, uint64_t* tot, size_t words, uint64_t max_body,
                                         const std::string& what) {
    exclusive_scan_u32(c, len, len, n, tot);
    std::vector<uint64_t> h = read_back<uint64_t>(c, tot, words);
    check_body(h[0], n, max_body, what);
    return h;
}

// rows [0, n) written at out + pos[r] by row_write_kernel, timed as `timer`; at most grid_per_sm blocks per SM
template <uint32_t STAGE, class R>
void row_write(Ctx* c, const R& rows, uint64_t n, const uint32_t* pos, uint8_t* out, const char* timer, uint64_t bytes, uint32_t grid_per_sm) {
    if (!n) return;
    KernelTimer kt(c, timer, bytes);
    constexpr uint32_t stages = ROW_WARPS * (STAGE + 16);
    CPB_CUDA(cudaFuncSetAttribute(row_write_kernel<R, STAGE>, cudaFuncAttributeMaxDynamicSharedMemorySize, stages + R::TABLE_BYTES));
    const uint32_t blocks = (uint32_t)std::min<uint64_t>((n + ROW_WARPS * 32 - 1) / (ROW_WARPS * 32), (uint64_t)c->sm_count * grid_per_sm);
    row_write_kernel<R, STAGE><<<blocks, ROW_WARPS * 32, stages + rows.tail(), c->stream>>>(rows, n, pos, out);
    CPB_CUDA(cudaGetLastError());
}

// ---- keyed columns: every column of a table with its name pre-encoded, in bytewise name order (strings.Compare, the
// order encoding/json gives map keys and WriteTo gives a row's pairs), as one device blob: KeyedCol[ncols], then the
// names at keys_at, meta_bytes in all.
struct KeyedCol {
    const uint32_t* off; const uint8_t* data;
    uint32_t key, key_len;  // the column's pre-encoded name in the name blob
};
struct KeyedCols { Buf md; uint32_t meta_bytes = 0, keys_at = 0; int ncols = 0; };
// (json.cu) the blob of t's columns from row lo on, uploaded without a host synchronisation; enc appends the encoding
// of the name of the k-th column in order.  keyed_value_bytes: *out = the value bytes of rows [0, n) of every column.
KeyedCols keyed_cols(Ctx* c, const Table& t, uint64_t lo, void (*enc)(std::string& keys, const std::string& name, int k));
void keyed_value_bytes(Ctx* c, const KeyedCols& kc, uint64_t n, unsigned long long* out);

// The base of the ToJSON and WriteTo row types: the blob, copied into shared memory when it fits in TABLE_BYTES, and
// row_const, the bytes every row has whatever its values.  Descriptors and names are contiguous in global memory as in
// shared.
struct KeyedRows {
    const KeyedCol* cols; const uint8_t* keys;
    int ncols;
    uint32_t meta_bytes;
    uint64_t row_const;
    KeyedRows(const KeyedCols& kc, uint64_t row_const)
        : cols(kc.md->as<KeyedCol>()), keys(kc.md->as<uint8_t>() + kc.keys_at), ncols(kc.ncols), meta_bytes(kc.meta_bytes), row_const(row_const) {}

    struct Tables { const KeyedCol* cols; const uint8_t* keys; };
    static constexpr uint32_t TABLE_BYTES = 16384;
    static constexpr bool TAIL_VARIES = true;
    uint32_t tail() const { return meta_bytes <= TABLE_BYTES ? meta_bytes : 0; }
    __device__ Tables stage(uint8_t* sm) const {
        if (meta_bytes > TABLE_BYTES) return {cols, keys};
        const uint8_t* gm = reinterpret_cast<const uint8_t*>(cols);
        for (uint32_t i = threadIdx.x; i < meta_bytes; i += blockDim.x) sm[i] = gm[i];
        __syncthreads();
        return {reinterpret_cast<const KeyedCol*>(sm), sm + (keys - gm)};
    }
};

}  // namespace cpb
