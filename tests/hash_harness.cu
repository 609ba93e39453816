// hash_harness.cu — the device's hashes of given inputs, computed by the functions the hash tables use, for
// tests/test_gpu_hash_collisions.py to compare with their restatement in tests/hash_ref.py:
//   keyhash.cuh: the value hash by one thread (hash_thread) and by a whole warp (hash_warp), GroupBy's row chain
//   (row_hash_step);
//   rowhash.cuh: pack3 of a KeyDesc, hash3, slot_of and hash_prefix.
//
//   hash_harness <in> <out>
// in (little-endian):
//   u64 nvals, u64 nbytes, nvals x {u64 off, u32 len, u32 k}, nbytes of value bytes
//     value i is bytes [off, off + len) of the bytes, so off % 8 is its start misalignment; k is its column in GroupBy's
//     row chain: the row of value i is values i - k .. i
//   u32 nkeys, u64 nrows, u64 nslots, u32 pbytes, u32 nwords,
//   per key column {u32 width, u32 lenbytes, u64 nbytes, u32 off[nrows + 1], nbytes of bytes},
//   u64 image[nwords][nrows]   (the key image, word-major as sort.cu lays it out)
// out:
//   per value {u64 thread hash, u64 warp hash, u64 row hash}
//   per key row {u64 w0, w1, w2 (pack3), hash3(w0, w1, w2), hash3(w0, w1, 0), slot_of of both in nslots, hash_prefix}
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "keyhash.cuh"
#include "rowhash.cuh"

using namespace cpb;

struct Val { uint64_t off; uint32_t len, k; };

__global__ void value_kernel(const Val* v, uint64_t n, const uint8_t* data, uint64_t* out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[3 * i] = hash_thread(data + v[i].off, v[i].len);
    uint64_t h = 0;
    for (uint32_t k = 0; k <= v[i].k; k++) {
        const Val& c = v[i - v[i].k + k];
        h = row_hash_step(h, hash_thread(data + c.off, c.len), k);
    }
    out[3 * i + 2] = h;
}
// one warp per value
__global__ void warp_kernel(const Val* v, uint64_t n, const uint8_t* data, uint64_t* out) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n) return;  // (whole warps)
    const uint64_t h = hash_warp(data + v[i].off, v[i].len, lane, 0, 0);
    if (lane == 0) out[3 * i + 1] = h;
}
__global__ void key_kernel(KeyDesc kd, uint64_t n, uint64_t nslots, const uint64_t* img, uint32_t pbytes, uint64_t* out) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    unsigned long long w0, w1, w2;
    pack3(kd, r, w0, w1, w2);
    const uint64_t h3 = hash3(w0, w1, w2), h2 = hash3(w0, w1, 0ull);
    uint64_t* o = out + 8 * r;
    o[0] = w0; o[1] = w1; o[2] = w2; o[3] = h3; o[4] = h2;
    o[5] = slot_of(h3, nslots); o[6] = slot_of(h2, nslots);
    o[7] = hash_prefix(img, n, r, pbytes);
}

static void check(cudaError_t e, const char* what) {
    if (e != cudaSuccess) { fprintf(stderr, "%s: %s\n", what, cudaGetErrorString(e)); exit(1); }
}
template <class T> static T get(FILE* f) {
    T x;
    if (fread(&x, sizeof x, 1, f) != 1) { fprintf(stderr, "short input\n"); exit(1); }
    return x;
}
template <class T> static std::vector<T> get_n(FILE* f, uint64_t n) {
    std::vector<T> v(n);
    if (n && fread(v.data(), sizeof(T), n, f) != n) { fprintf(stderr, "short input\n"); exit(1); }
    return v;
}
// a device copy of v, padded with 16 zero bytes (word_at and load16 read whole aligned words)
template <class T> static T* upload(const std::vector<T>& v) {
    void* p = nullptr;
    const size_t b = v.size() * sizeof(T);
    check(cudaMalloc(&p, b + 16), "cudaMalloc");
    check(cudaMemset(p, 0, b + 16), "cudaMemset");
    if (b) check(cudaMemcpy(p, v.data(), b, cudaMemcpyHostToDevice), "upload");
    return (T*)p;
}

int main(int argc, char** argv) {
    if (argc != 3) { fprintf(stderr, "usage: hash_harness <in> <out>\n"); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { perror(argv[1]); return 1; }
    const uint64_t nv = get<uint64_t>(f), nb = get<uint64_t>(f);
    const std::vector<Val> vals = get_n<Val>(f, nv);
    const std::vector<uint8_t> bytes = get_n<uint8_t>(f, nb);
    KeyDesc kd{};
    kd.nkeys = (int)get<uint32_t>(f);
    const uint64_t nr = get<uint64_t>(f), nslots = get<uint64_t>(f);
    const uint32_t pbytes = get<uint32_t>(f);
    kd.words = get<uint32_t>(f);
    for (int k = 0; k < kd.nkeys; k++) {
        kd.width[k] = get<uint32_t>(f);
        kd.lenbytes[k] = get<uint32_t>(f);
        const uint64_t kb = get<uint64_t>(f);
        kd.off[k] = upload(get_n<uint32_t>(f, nr + 1));
        kd.data[k] = upload(get_n<uint8_t>(f, kb));
    }
    const uint64_t* img = upload(get_n<uint64_t>(f, (uint64_t)kd.words * nr));
    fclose(f);

    std::vector<uint64_t> vout(3 * nv), kout(8 * nr);
    uint64_t* dv = upload(vout);
    uint64_t* dk = upload(kout);
    if (nv) {
        const Val* v = upload(vals);
        const uint8_t* d = upload(bytes);
        value_kernel<<<(unsigned)((nv + 255) / 256), 256>>>(v, nv, d, dv);
        warp_kernel<<<(unsigned)((nv * 32 + 255) / 256), 256>>>(v, nv, d, dv);
    }
    if (nr) key_kernel<<<(unsigned)((nr + 255) / 256), 256>>>(kd, nr, nslots, img, pbytes, dk);
    check(cudaGetLastError(), "launch");
    check(cudaDeviceSynchronize(), "kernels");
    check(cudaMemcpy(vout.data(), dv, vout.size() * 8, cudaMemcpyDeviceToHost), "download");
    check(cudaMemcpy(kout.data(), dk, kout.size() * 8, cudaMemcpyDeviceToHost), "download");
    FILE* o = fopen(argv[2], "wb");
    if (!o) { perror(argv[2]); return 1; }
    fwrite(vout.data(), 8, vout.size(), o);
    fwrite(kout.data(), 8, kout.size(), o);
    fclose(o);
    return 0;
}
