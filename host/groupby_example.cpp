// groupby_example.cpp — per-customer aggregates through the C++ mirror (host/csvplus.hpp, DataSource::GroupBy): the qty
// sums of TestSimpleUniqueJoin (csvplus_test.go:368-452) after a join with the customers' unique index, and the amounts
// of TestTransformedSource (:754-806), amount = FormatFloat(price * qty, 'f', 2) summed per customer as
// custAmounts[cid] += amount does.  Both are checked against the same folds on the host, the float sums bit for bit.
// Exit code 0 = all checks hold.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <map>
#include <vector>

#include "csvplus.hpp"

using namespace csvplus;

#define CHECK(c) do { if (!(c)) { fprintf(stderr, "CHECK failed %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

int main() {
    std::string people = "id,name,surname\n";
    for (int i = 0; i < 120; i++) people += std::to_string(i) + ",N" + std::to_string(i % 10) + ",S" + std::to_string(i % 12) + "\n";
    const double price[] = {0.99, 12.5, 3.3, 7.15, 100.01, 0.1, 42.0, 5.55};
    std::string orders = "order_id,cust_id,prod_id,qty\n";
    std::vector<int> cust(20000), prod(20000), qty(20000);
    unsigned s = 12345;
    for (int i = 0; i < 20000; i++) {
        s = s * 1103515245u + 12345u; cust[i] = (s >> 8) % 130;  // ids 120..129 have no customer: the join drops them
        s = s * 1103515245u + 12345u; qty[i] = 1 + (s >> 8) % 100;
        prod[i] = i % 8;
        orders += std::to_string(i) + "," + std::to_string(cust[i]) + "," + std::to_string(prod[i]) + "," + std::to_string(qty[i]) + "\n";
    }
    try {
        // TestSimpleUniqueJoin: sum(qty) per customer of the joined rows
        Index idx = Take(FromString(people)).UniqueIndexOn({"id"});
        Groups q = Take(FromString(orders).SelectColumns({"order_id", "cust_id", "qty"})).Join(idx, {"cust_id"})
                       .GroupBy({"cust_id"}, {{"qty", CPB_AGG_SUM, "qty", CPB_AGG_INT}, {"orders", CPB_AGG_COUNT, ""}});
        std::map<std::string, int64_t> want_qty, want_n;
        std::vector<std::string> first_seen;
        for (int i = 0; i < 20000; i++) {
            if (cust[i] >= 120) continue;
            const std::string k = std::to_string(cust[i]);
            if (!want_n.count(k)) first_seen.push_back(k);
            want_qty[k] += qty[i];
            want_n[k]++;
        }
        const uint64_t n = q.size();
        CHECK(n == first_seen.size());
        std::vector<int64_t> got_qty(n), got_n(n);
        CHECK(cpb_memcpy_d2h(detail::ctx(), got_qty.data(), q.Int("qty"), n * 8) == CPB_OK);
        CHECK(cpb_memcpy_d2h(detail::ctx(), got_n.data(), q.Int("orders"), n * 8) == CPB_OK);
        std::vector<Row> keys = q.Keys().rows();
        CHECK(keys.size() == n);
        for (uint64_t g = 0; g < n; g++) {
            CHECK(keys[g].at("cust_id") == first_seen[g]);
            CHECK(got_qty[g] == want_qty[first_seen[g]] && got_n[g] == want_n[first_seen[g]]);
        }

        // TestTransformedSource: amount = FormatFloat(price * qty, 'f', 2), custAmounts[cid] += amount
        auto amount = [&](const Row& r) {
            Row o = r;
            char buf[64];
            snprintf(buf, sizeof buf, "%.2f", price[std::stoi(r.at("prod_id"))] * std::stod(r.at("qty")));
            o["amount"] = buf;
            return o;
        };
        Groups a = Take(FromString(orders)).Map(amount).GroupBy({"cust_id"}, {{"amount", CPB_AGG_SUM, "amount", CPB_AGG_FLOAT64}});
        std::map<std::string, double> want_amt;
        std::vector<std::string> order;
        for (int i = 0; i < 20000; i++) {
            const std::string k = std::to_string(cust[i]);
            char buf[64];
            snprintf(buf, sizeof buf, "%.2f", price[prod[i]] * (double)qty[i]);
            if (!want_amt.count(k)) { order.push_back(k); want_amt[k] = 0.0; }
            want_amt[k] += strtod(buf, nullptr);
        }
        CHECK(a.size() == order.size());
        std::vector<double> got_amt(a.size());
        CHECK(cpb_memcpy_d2h(detail::ctx(), got_amt.data(), a.Float64("amount"), a.size() * 8) == CPB_OK);
        std::vector<Row> akeys = a.Keys().rows();
        for (size_t g = 0; g < order.size(); g++) {
            const double w = want_amt[order[g]];
            CHECK(akeys[g].at("cust_id") == order[g] && memcmp(&got_amt[g], &w, 8) == 0);
        }
        std::cout << "groupby example ok: " << n << " customers joined, " << a.size() << " customers with amounts\n";
    } catch (const std::exception& e) {
        std::cerr << "error: " << e.what() << "\n";
        return 1;
    }
    return 0;
}
