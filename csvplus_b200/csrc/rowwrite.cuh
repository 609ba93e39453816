// rowwrite.cuh — what the row serialisers share: the warp-staged row writer of ToCsv (write.cu), ToJSON (json.cu),
// Index.WriteTo (gob.cu) and FormatInt / FormatFloat (format.cu), and the keyed-column table of ToJSON and WriteTo.
#pragma once
#include "core.hpp"

namespace cpb {

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
    uint8_t* stage = stages + warp * (int)(STAGE + 16);  // signed: with an unsigned offset ptxas spills in json_write
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

// The block copies the blob into shared memory at sm when meta_smem, and cols / keys then point there; else they keep
// pointing into global memory.  Descriptors and names are contiguous in global memory as in shared.
__device__ __forceinline__ void stage_keyed_cols(uint8_t* sm, int meta_smem, uint32_t meta_bytes, const KeyedCol*& cols, const uint8_t*& keys) {
    if (!meta_smem) return;
    const uint8_t* gm = reinterpret_cast<const uint8_t*>(cols);
    for (uint32_t i = threadIdx.x; i < meta_bytes; i += blockDim.x) sm[i] = gm[i];
    __syncthreads();
    cols = reinterpret_cast<const KeyedCol*>(sm);
    keys = sm + (keys - gm);
}

}  // namespace cpb
