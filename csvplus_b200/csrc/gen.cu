// gen.cu — deterministic synthetic CSV generators (bench / test infrastructure, not part of the
// product path).  Shapes follow SURVEY §8(d), which in turn follow the reference's own fixture
// generators (csvplus_test.go:1207-1333): people/customers, orders, products.  Every field is a
// pure function of (seed, table, row, column) through splitmix64, so any row range can be produced
// independently on any GPU.
#include "core.hpp"
#include "util.cuh"

namespace cpb {

struct GenParams {
    int kind;  // 0 people/customers, 1 orders, 2 products
    uint64_t seed, row_lo, row_hi, n_cust, n_prod;
    uint64_t perm_a, perm_b, perm_n;  // id = (a*row + b) mod n when perm_n != 0
    uint32_t header_len;
};

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
__device__ __forceinline__ uint64_t rnd(const GenParams& g, uint64_t row, uint32_t col) {
    return splitmix64(g.seed ^ ((uint64_t)(g.kind + 1) << 56) ^ (row * 0xD1342543DE82EF95ull) ^ ((uint64_t)col * 0xA24BAED4963EE407ull));
}

__constant__ char c_names[10][8] = {"Amelia", "Olivia", "Emily", "Ava", "Isla", "Oliver", "Jack", "Harry", "Jacob", "Charlie"};
__constant__ char c_surnames[12][10] = {"Smith", "Jones", "Taylor", "Williams", "Brown", "Davies",
                                        "Evans", "Wilson", "Thomas", "Roberts", "Johnson", "Lewis"};
__constant__ char c_cities[16][12] = {"London", "Leeds", "Bristol", "Glasgow", "Cardiff", "Belfast", "Liverpool", "Manchester",
                                      "Sheffield", "Edinburgh", "Oxford", "York", "Bath", "Derby", "Hull", "Exeter"};

struct Emit {  // counts, or writes when p != nullptr
    uint8_t* p; uint32_t n = 0;
    __device__ void ch(char c) { if (p) p[n] = (uint8_t)c; n++; }
    __device__ void str(const char* s) { while (*s) ch(*s++); }
    __device__ void num(uint64_t v) {
        char b[20]; int k = 0;
        do { b[k++] = (char)('0' + v % 10); v /= 10; } while (v);
        while (k) ch(b[--k]);
    }
    __device__ void num_pad(uint64_t v, int width) {
        char b[20]; int k = 0;
        do { b[k++] = (char)('0' + v % 10); v /= 10; } while (v);
        for (int i = k; i < width; i++) ch('0');
        while (k) ch(b[--k]);
    }
};

__device__ void emit_row(const GenParams& g, uint64_t row, Emit& e) {
    uint64_t id = g.perm_n ? (g.perm_a * row + g.perm_b) % g.perm_n : row;
    if (g.kind == 0) {  // id,name,surname,born,city,score
        e.num(id); e.ch(',');
        e.str(c_names[rnd(g, row, 1) % 10]); e.ch(',');
        e.str(c_surnames[rnd(g, row, 2) % 12]); e.ch(',');
        e.num(1916 + rnd(g, row, 3) % 90); e.ch(',');
        e.str(c_cities[rnd(g, row, 4) % 16]); e.ch(',');
        uint64_t s = rnd(g, row, 5);
        e.num(s % 100000); e.ch('.'); e.num_pad((s >> 32) % 100, 2);
    } else if (g.kind == 1) {  // order_id,cust_id,prod_id,qty,ts
        e.num(row); e.ch(',');
        e.num(rnd(g, row, 1) % g.n_cust); e.ch(',');
        e.num(rnd(g, row, 2) % g.n_prod); e.ch(',');
        e.num(1 + rnd(g, row, 3) % 100); e.ch(',');
        // RFC3339 with +01:00 zone: 2016-09-14T08:48:22+01:00 minus u[1,1e5] seconds
        int64_t t = 1473839302ll + 3600 - (int64_t)(1 + rnd(g, row, 4) % 100000);
        int64_t days = t / 86400, rem = t % 86400;
        int64_t z = days + 719468, era = z / 146097, doe = z - era * 146097;
        int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365, y = yoe + era * 400;
        int64_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100), mp = (5 * doy + 2) / 153;
        int64_t d = doy - (153 * mp + 2) / 5 + 1, m = mp < 10 ? mp + 3 : mp - 9;
        if (m <= 2) y++;
        e.num_pad((uint64_t)y, 4); e.ch('-'); e.num_pad((uint64_t)m, 2); e.ch('-'); e.num_pad((uint64_t)d, 2); e.ch('T');
        e.num_pad((uint64_t)(rem / 3600), 2); e.ch(':'); e.num_pad((uint64_t)(rem % 3600 / 60), 2); e.ch(':'); e.num_pad((uint64_t)(rem % 60), 2);
        e.str("+01:00");
    } else {  // prod_id,product,price
        e.num(id); e.ch(',');
        e.str("item"); e.num_pad(id, 7); e.ch(',');
        uint64_t s = rnd(g, row, 2);
        e.num(s % 1000); e.ch('.'); e.num_pad((s >> 32) % 100, 2);
    }
    e.ch('\n');
}

static void gen_lengths(Ctx* c, const GenParams& g, uint32_t* len) {
    each_row(c, g.row_hi - g.row_lo, [=] __device__(uint64_t i) {
        Emit e{nullptr};
        emit_row(g, g.row_lo + i, e);
        len[i] = e.n;
    });
}
// the rows at dst + header_len + off[i] (off: the scanned lengths)
static void gen_write(Ctx* c, const GenParams& g, const uint32_t* off, uint8_t* dst) {
    uint8_t* body = dst + g.header_len;
    each_row(c, g.row_hi - g.row_lo, [=] __device__(uint64_t i) {
        Emit e{body + off[i]};
        emit_row(g, g.row_lo + i, e);
    });
}

}  // namespace cpb

using namespace cpb;

static uint64_t gcd64(uint64_t a, uint64_t b) { while (b) { uint64_t t = a % b; a = b; b = t; } return a; }

extern "C" int cpb_gen_csv(cpb_ctx* h, int kind, uint64_t seed, uint64_t row_lo, uint64_t row_hi, uint64_t n_cust, uint64_t n_prod,
                           int with_header, int permute, void* dst, uint64_t cap, uint64_t* nbytes) {
    return guarded(h, nullptr, [&](Ctx* c) {
        need(nbytes, "null nbytes");
        if (kind < 0 || kind > 2 || row_hi < row_lo) throw ArgError{CPB_ERR_ARG, "bad generator arguments"};
        static const char* headers[3] = {"id,name,surname,born,city,score\n", "order_id,cust_id,prod_id,qty,ts\n", "prod_id,product,price\n"};
        GenParams gp{};
        gp.kind = kind; gp.seed = seed; gp.row_lo = row_lo; gp.row_hi = row_hi; gp.n_cust = n_cust ? n_cust : 1; gp.n_prod = n_prod ? n_prod : 1;
        gp.header_len = with_header ? (uint32_t)strlen(headers[kind]) : 0;
        if (permute) {
            uint64_t n = kind == 2 ? gp.n_prod : gp.n_cust;  // ids are a bijection of [0, table size)
            uint64_t a = (0x9E3779B97F4A7C15ull ^ seed) % n;
            if (a < 2) a = n > 2 ? 2 : 1;
            while (gcd64(a, n) != 1) a++;
            gp.perm_a = a % n; gp.perm_b = (seed * 0x2545F4914F6CDD1Dull) % n; gp.perm_n = n;
            if (n >= (1ull << 32)) throw ArgError{CPB_ERR_ARG, "permuted tables are limited to 2^32 rows"};
        }
        const uint64_t rows = row_hi - row_lo;
        Buf len = dev_alloc(c, (rows + 1) * 4), total = dev_alloc(c, 8);
        gen_lengths(c, gp, len->as<uint32_t>());
        exclusive_scan_u32(c, len->as<uint32_t>(), len->as<uint32_t>(), rows, total->as<uint64_t>());
        const uint64_t body = read_back<uint64_t>(c, total->p);
        if (body > 0xffffffffull) throw ArgError{CPB_ERR_ARG, "generate at most 4 GiB per call (split the row range)"};
        *nbytes = body + gp.header_len;
        if (dst) {
            if (*nbytes > cap) throw ArgError{CPB_ERR_ARG, "generator destination too small"};
            if (gp.header_len) CPB_CUDA(cudaMemcpyAsync(dst, headers[kind], gp.header_len, cudaMemcpyHostToDevice, c->stream));
            gen_write(c, gp, len->as<uint32_t>(), (uint8_t*)dst);
            sync_stream(c);
        }
        return CPB_OK;
    });
}
