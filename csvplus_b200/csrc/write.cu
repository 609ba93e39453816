// write.cu — K10 of SURVEY §2: DataSource.ToCsv (csvplus.go:379-406) with the default
// encoding/csv.Writer (comma ',', UseCRLF=false; SURVEY App. B): header line, then one line per row
// with the named columns in caller order.  A field is quoted iff it is non-empty and (it is `\.` or
// contains , " \r \n or its first rune is unicode.IsSpace); inside quotes " is doubled.
// The row type CsvRows through the row serialiser driver of rowwrite.cuh.
#include "core.hpp"
#include "rowwrite.cuh"

namespace cpb {

constexpr int MAXW = 64;  // columns per ToCsv call

__host__ __device__ inline bool first_rune_is_space(const uint8_t* p, uint32_t n) {
    uint8_t c = p[0];
    if (c < 0x80) return c == ' ' || (c >= '\t' && c <= '\r');
    if (c == 0xC2 && n >= 2) return p[1] == 0x85 || p[1] == 0xA0;
    if (c == 0xE1 && n >= 3) return p[1] == 0x9A && p[2] == 0x80;
    if (c == 0xE2 && n >= 3) {
        if (p[1] == 0x80) return (p[2] >= 0x80 && p[2] <= 0x8A) || p[2] == 0xA8 || p[2] == 0xA9 || p[2] == 0xAF;
        return p[1] == 0x81 && p[2] == 0x9F;
    }
    if (c == 0xE3 && n >= 3) return p[1] == 0x80 && p[2] == 0x80;
    return false;
}
// returns output length of one field (up to 2n + 2, so 64 bits); *quoted tells whether it is written in quotes
__host__ __device__ inline uint64_t field_out_len(const uint8_t* p, uint32_t n, bool* quoted) {
    *quoted = false;
    if (n == 0) return 0;
    uint32_t nq = 0; bool need = (n == 2 && p[0] == '\\' && p[1] == '.');
    for (uint32_t i = 0; i < n; i++) {
        uint8_t c = p[i];
        if (c == '"') { nq++; need = true; }
        else if (c == ',' || c == '\r' || c == '\n') need = true;
    }
    if (!need) need = first_rune_is_space(p, n);
    *quoted = need;
    return need ? (uint64_t)n + nq + 2 : n;
}
__host__ __device__ inline uint32_t field_write(const uint8_t* p, uint32_t n, uint8_t* d) {
    bool q; field_out_len(p, n, &q);
    if (!q) { for (uint32_t i = 0; i < n; i++) d[i] = p[i]; return n; }
    uint32_t k = 0;
    d[k++] = '"';
    for (uint32_t i = 0; i < n; i++) { if (p[i] == '"') d[k++] = '"'; d[k++] = p[i]; }
    d[k++] = '"';
    return k;
}

// a row: the named columns in caller order, each field through the quoting rule, then '\n'.  A row of quotes doubles
// in length, and a column may be named more than once.
struct CsvRows : NoTables {
    int n; const uint32_t* off[MAXW]; const uint8_t* data[MAXW];
    __device__ uint64_t len(uint64_t r) const {
        uint64_t total = (uint64_t)n;  // n-1 commas + newline
        for (int k = 0; k < n; k++) {
            const uint32_t s = off[k][r], l = off[k][r + 1] - s;
            bool q;
            total += field_out_len(data[k] + s, l, &q);
        }
        return total;
    }
    __device__ void write(uint64_t r, uint8_t* q, Tables) const {
        for (int k = 0; k < n; k++) {
            if (k) *q++ = ',';
            const uint32_t s = off[k][r], l = off[k][r + 1] - s;
            q += field_write(data[k] + s, l, q);
        }
        *q = '\n';
    }
};

Buf table_to_csv(Ctx* c, const Table& t, const std::vector<int>& cols, const std::vector<std::string>& names, bool with_header,
                 uint64_t room, uint64_t* nbytes) {
    if ((int)cols.size() > MAXW) throw ArgError{CPB_ERR_UNSUPPORTED, "more than 64 columns in ToCsv"};
    // header line (csvplus.go:387): the caller's column names through the same quoting rule
    std::string header;
    for (size_t i = 0; with_header && i < names.size(); i++) {
        if (i) header += ',';
        std::vector<uint8_t> tmp(names[i].size() * 2 + 2);
        uint32_t k = field_write((const uint8_t*)names[i].data(), (uint32_t)names[i].size(), tmp.data());
        header.append((const char*)tmp.data(), k);
    }
    if (with_header) header += '\n';
    const uint64_t n = (uint64_t)t.nrows;
    CsvRows rows{};
    rows.n = (int)cols.size();
    for (int k = 0; k < rows.n && n; k++) { rows.off[k] = t.cols[cols[k]].off(); rows.data[k] = t.cols[cols[k]].bytes(); }
    Buf len = dev_alloc(c, (n + 1) * 4), tot = dev_alloc(c, 8);
    row_lengths(c, rows, n, len->as<uint32_t>(), "csv_row_len", n * 4 * (rows.n + 1));
    const uint64_t body = row_offsets(c, len->as<uint32_t>(), n, tot->as<uint64_t>(), 1, MAX_BODY,
                                      "ToCsv output exceeds 4 GiB; write in smaller batches")[0];
    *nbytes = header.size() + body;
    if (*nbytes > room) return nullptr;
    Buf out = dev_alloc(c, header.size() + body + 16);
    CPB_CUDA(cudaMemcpyAsync(out->p, header.data(), header.size(), cudaMemcpyHostToDevice, c->stream));
    row_write<4096>(c, rows, n, len->as<uint32_t>(), out->as<uint8_t>() + header.size(), "csv_write", 2 * body + n * 4 * (rows.n + 1), 16);
    return out;
}

}  // namespace cpb
