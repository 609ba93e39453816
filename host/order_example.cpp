// order_example.cpp — ORDER BY price DESC LIMIT 10 through the C++ mirror (host/csvplus.hpp, DataSource::OrderBy): the ten
// most expensive orders of a file read in many batches, folded batch by batch on the GPU.  Checked against
// std::stable_sort of the same rows on the host with cmp.Compare(b, a) on the prices (NaNs last, ties in file order), and
// against the materialised order (OrderBy, then SelectColumns, then Top).  Exit code 0 = all checks hold.
#include <unistd.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "csvplus.hpp"

using namespace csvplus;

#define CHECK(c) do { if (!(c)) { fprintf(stderr, "CHECK failed %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

int main() {
    const int n = 200000;
    std::string csv = "id,cust_id,price\n";
    std::vector<double> price(n);
    std::vector<std::string> text(n);
    unsigned s = 777;
    for (int i = 0; i < n; i++) {
        s = s * 1103515245u + 12345u;
        text[i] = i % 1000 == 7 ? "NaN" : std::to_string((s >> 8) % 5000) + "." + std::to_string((s >> 4) % 10) + "5";
        price[i] = strtod(text[i].c_str(), nullptr);
        csv += std::to_string(i) + ",c" + std::to_string(i % 97) + "," + text[i] + "\n";
    }
    const char* dir = getenv("TMPDIR");
    std::string name = std::string(dir && *dir ? dir : "/tmp") + "/order_example_XXXXXX";
    const int fd = mkstemp(&name[0]);
    CHECK(fd >= 0);
    CHECK(write(fd, csv.data(), csv.size()) == (ssize_t)csv.size());
    close(fd);
    int rc = 0;
    try {
        // cmp.Compare(price[b], price[a]) in a stable sort: descending, NaNs last, ties in file order
        std::vector<int> want(n);
        for (int i = 0; i < n; i++) want[i] = i;
        std::stable_sort(want.begin(), want.end(), [&](int a, int b) {
            const double x = price[a], y = price[b];
            if (std::isnan(x) || std::isnan(y)) return std::isnan(y) && !std::isnan(x);
            return x > y;
        });
        StreamBatchBytes() = 64 << 10;  // about 60 batches
        const std::vector<OrderKey> by_price{{"price", CPB_ORDER_FLOAT64, true}};
        std::vector<Row> top = Take(FromFile(name)).OrderBy(by_price).Top(10).ToRows();
        std::vector<Row> whole = Take(FromFile(name)).OrderBy(by_price).SelectColumns({"id", "cust_id", "price"}).Top(10).ToRows();
        CHECK(top.size() == 10 && whole.size() == 10);
        for (int i = 0; i < 10; i++) {
            CHECK(top[i]["id"] == std::to_string(want[i]));
            CHECK(top[i] == whole[i]);
            printf("%s,%s\n", top[i]["id"].c_str(), top[i]["price"].c_str());
        }
        // Table::OrderBy: the last rows of the ascending order are the NaNs, in file order
        Table t = Take(FromFile(name)).ToTable();
        Table asc = t.OrderBy({{"price", CPB_ORDER_FLOAT64}, {"id", CPB_ORDER_INT}}, 3);
        std::vector<Row> first = asc.rows();
        CHECK(first.size() == 3 && first[0]["price"] == "NaN" && first[0]["id"] == "7" && first[2]["id"] == "2007");
        // a failing conversion is an Error
        bool threw = false;
        try { Take(FromFile(name)).OrderBy({{"cust_id", CPB_ORDER_INT}}).Top(1).ToRows(); } catch (const Error& e) { threw = std::string(e.what()).find("cannot convert") != std::string::npos; }
        CHECK(threw);
        printf("order example ok\n");
    } catch (const std::exception& e) {
        fprintf(stderr, "error: %s\n", e.what());
        rc = 1;
    }
    unlink(name.c_str());
    return rc;
}
