// format_example.cpp — the reference's createAmountsTable (csvplus_test.go:1391-1421) through the C++ mirror
// (host/csvplus.hpp): orders joined with a stock index, qty and price converted on the GPU (ValuesAsInt /
// ValuesAsFloat64), the product computed on the host, then row["amount"] = strconv.FormatFloat(price*qty, 'f', 2, 64)
// set on the GPU (Table::WithColumn), price and qty dropped, and the rows written to stdout as CSV.
#include <iostream>
#include <vector>

#include "csvplus.hpp"

using namespace csvplus;

int main() {
    std::string orders = "cust_id,prod_id,qty\n", stock = "prod_id,price\n";
    for (int i = 0; i < 1000; i++)
        orders += std::to_string(i) + "," + std::to_string(i % 50) + "," + std::to_string(i % 13 - 3) + "\n";
    for (int p = 0; p < 50; p++) stock += std::to_string(p) + "," + std::to_string(p * 1.25 + 0.5) + "\n";
    Index prod = Take(FromString(stock).SelectColumns({"prod_id", "price"})).UniqueIndexOn({"prod_id"});
    Table t = Take(FromString(orders).SelectColumns({"cust_id", "prod_id", "qty"})).Join(prod).ToTable();
    const size_t n = (size_t)t.size();
    cpb_ctx* ctx = detail::ctx();
    void *dq = nullptr, *dpr = nullptr;
    if (cpb_device_alloc(ctx, n * 8 + 8, &dq) != CPB_OK || cpb_device_alloc(ctx, n * 8 + 8, &dpr) != CPB_OK) throw Error(cpb_last_error(ctx));
    t.ValuesAsInt("qty", (int64_t*)dq);
    t.ValuesAsFloat64("price", (double*)dpr);
    std::vector<int64_t> qty(n);
    std::vector<double> price(n);
    if (cpb_memcpy_d2h(ctx, qty.data(), dq, n * 8) != CPB_OK || cpb_memcpy_d2h(ctx, price.data(), dpr, n * 8) != CPB_OK) throw Error(cpb_last_error(ctx));
    for (size_t i = 0; i < n; i++) price[i] *= (double)qty[i];
    if (cpb_memcpy_h2d(ctx, dpr, price.data(), n * 8) != CPB_OK) throw Error(cpb_last_error(ctx));
    Table amounts = t.WithColumn("amount", (const double*)dpr, 'f', 2);
    DataSource(amounts).DropColumns({"price", "qty"}).ToCsv(std::cout, {"cust_id", "prod_id", "amount"});
    cpb_device_free(ctx, dq);
    cpb_device_free(ctx, dpr);
    return 0;
}
