// float32_example.cpp — float32 columns through the C++ mirror (host/csvplus.hpp): a column of decimal strings read
// as float values on the GPU (Table::ValuesAsFloat32, strconv.ParseFloat(s, 32)), written back as two new columns
// with strconv.FormatFloat(float64(x), 'g', -1, 32) and FormatFloat(float64(x), 'f', 2, 32) (Table::WithColumn of
// float values), the rows written to stdout as CSV.  Then a value out of float32's range: the error line it throws.
#include <iostream>

#include "csvplus.hpp"

using namespace csvplus;

int main() {
    std::string csv = "s\n0.1\n1.00000005960464477539062500000001\n16777217\n3.4028235e38\n1e-45\n-0\n";
    for (int i = 0; i < 1000; i++) csv += std::to_string(i * 37 % 1000) + "." + std::to_string(i % 100) + "e" + std::to_string(i % 61 - 30) + "\n";
    Table t = Take(FromString(csv)).ToTable();
    const size_t n = (size_t)t.size();
    cpb_ctx* ctx = detail::ctx();
    void* dv = nullptr;
    if (cpb_device_alloc(ctx, n * 4 + 4, &dv) != CPB_OK) throw Error(cpb_last_error(ctx));
    t.ValuesAsFloat32("s", (float*)dv);
    Table out = t.WithColumn("g", (const float*)dv, 'g', -1).WithColumn("f2", (const float*)dv, 'f', 2);
    DataSource(out).ToCsv(std::cout, {"s", "g", "f2"});
    cpb_device_free(ctx, dv);
    Table big = Take(FromString("s\n1\n1e39\n")).ToTable();
    if (cpb_device_alloc(ctx, 8, &dv) != CPB_OK) throw Error(cpb_last_error(ctx));
    try {
        big.ValuesAsFloat32("s", (float*)dv);
        std::cout << "no error\n";
    } catch (const Error& e) {
        std::cout << "error: " << e.what() << "\n";
    }
    cpb_device_free(ctx, dv);
    return 0;
}
