// codes_example.cpp — categorical codes through the C++ mirror (host/csvplus.hpp): a string column with quoted commas,
// empty values and values of 5000 bytes encoded on the GPU (Table::ValuesAsCodes), the codes and the dictionary
// written to stdout, the column rebuilt from the codes (Table::WithColumn of codes and a dictionary) and compared with
// the original, then a code outside the dictionary: the error line it throws.
#include <iostream>
#include <vector>

#include "csvplus.hpp"

using namespace csvplus;

int main() {
    const std::string vals[] = {"red", "", "\"a,b\"", "green", std::string(5000, 'x') + "1", std::string(5000, 'x') + "2", "re"};
    std::string csv = "id,name\n";
    for (int i = 0; i < 3000; i++) csv += std::to_string(i) + "," + vals[(i * i + 3 * i) % 7 % (i < 5 ? 3 : 7)] + "\n";
    Table t = Take(FromString(csv)).ToTable();
    const size_t n = (size_t)t.size();
    cpb_ctx* ctx = detail::ctx();
    void* dv = nullptr;
    if (cpb_device_alloc(ctx, n * 8 + 8, &dv) != CPB_OK) throw Error(cpb_last_error(ctx));
    Table dict = t.ValuesAsCodes("name", (int64_t*)dv);
    std::vector<int64_t> codes(n);
    if (cpb_memcpy_d2h(ctx, codes.data(), dv, n * 8) != CPB_OK) throw Error(cpb_last_error(ctx));
    std::cout << "rows " << n << " distinct " << dict.size() << "\n";
    for (size_t i = 0; i < n; i++) std::cout << codes[i] << (i + 1 < n ? " " : "\n");
    DataSource(dict).ToCsv(std::cout, {"name"});
    Table back = t.WithColumn("back", (const int64_t*)dv, dict);
    size_t same = 0;
    for (const Row& r : back.rows()) same += r.at("back") == r.at("name");
    std::cout << "round trip " << same << " of " << n << "\n";
    codes[n - 1] = dict.size();
    if (cpb_memcpy_h2d(ctx, dv, codes.data(), n * 8) != CPB_OK) throw Error(cpb_last_error(ctx));
    try {
        t.WithColumn("name", (const int64_t*)dv, dict);
        std::cout << "no error\n";
    } catch (const Error& e) {
        std::cout << "error: " << e.what() << "\n";
    }
    cpb_device_free(ctx, dv);
    return 0;
}
