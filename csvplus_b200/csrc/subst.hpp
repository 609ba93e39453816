// subst.hpp — stand-in bytes for multi-byte reader runes (subst.cu)
#pragma once
#include "core.hpp"

namespace cpb {

constexpr int MAX_SUB_SEQ = 24;
// device-visible expansion table: byte value -> the UTF-8 sequence it stands for (len 0 = an ordinary byte)
struct SubTable {
    uint32_t bits[8];        // stand-in bytes
    uint32_t space_bits[8];  // those standing for a Unicode space (TrimLeadingSpace trims them at a field start)
    uint8_t len[256];
    uint8_t seq[256][4];
};
__host__ __device__ inline bool sub_is(const uint32_t* bits, int c) { return c >= 0 && ((bits[(c >> 5) & 7] >> (c & 31)) & 1u) != 0; }

struct Substitution {
    Buf buffer;             // transcoded input (null: the original input is parsed)
    uint64_t nbytes = 0;
    uint32_t delimiter = 0, comment = 0;  // single-byte values for the kernels
    Buf table;              // SubTable in device memory (null: no stand-ins)
    SubTable host_table{};
};
bool needs_substitution(const cpb_reader_opts& o);
std::string utf8_rune(uint32_t r);
// the multi-byte runes unicode.IsSpace accepts: what TrimLeadingSpace trims besides ASCII white space
constexpr uint32_t kUnicodeSpaces[] = {0x85, 0xA0, 0x1680, 0x2000, 0x2001, 0x2002, 0x2003, 0x2004, 0x2005, 0x2006,
                                       0x2007, 0x2008, 0x2009, 0x200A, 0x2028, 0x2029, 0x202F, 0x205F, 0x3000};
Substitution substitute_runes(Ctx* c, const uint8_t* in, uint64_t n, const cpb_reader_opts& o);

}  // namespace cpb
