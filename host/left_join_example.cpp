// left_join_example.cpp — every order enriched with its customer and product where they are known, through the C++ mirror
// (host/csvplus.hpp, DataSource::LeftJoin): orders whose customer or product is missing from the indexes are kept, with
// the customer's / product's columns empty.  Read in many batches.  Checked against a host loop over std::map lookups
// (Row.SafeGetValue(col, "") on a miss), and the matched rows against Join.  Exit code 0 = all checks hold.
#include <cstdio>
#include <map>
#include <string>
#include <vector>

#include "csvplus.hpp"

using namespace csvplus;

#define CHECK(c) do { if (!(c)) { fprintf(stderr, "CHECK failed %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

int main() {
    const int ncust = 900, nprod = 40, nord = 50000;
    std::string customers = "id,name\n", products = "prod_id,price\n", orders = "order_id,cust_id,prod_id,qty\n";
    std::map<std::string, std::string> name, price;
    for (int i = 0; i < ncust; i++) {
        const std::string id = "c" + std::to_string(i), nm = "name" + std::to_string(i * 7 % 1000);
        customers += id + "," + nm + "\n";
        name[id] = nm;
    }
    for (int i = 0; i < nprod; i++) {
        const std::string id = "p" + std::to_string(i), pr = std::to_string(i) + ".25";
        products += id + "," + pr + "\n";
        price[id] = pr;
    }
    std::vector<std::vector<std::string>> ord;
    unsigned s = 4242;
    for (int i = 0; i < nord; i++) {  // customer ids up to 999 and product ids up to 44: about 10 % unknown of each
        s = s * 1103515245u + 12345u;
        ord.push_back({std::to_string(i), "c" + std::to_string((s >> 8) % 1000), "p" + std::to_string((s >> 4) % 45),
                       std::to_string((s >> 12) % 9 + 1)});
        orders += ord.back()[0] + "," + ord.back()[1] + "," + ord.back()[2] + "," + ord.back()[3] + "\n";
    }
    try {
        Index cust = Take(FromString(customers)).UniqueIndexOn({"id"});
        Index prod = Take(FromString(products)).UniqueIndexOn({"prod_id"});
        StreamBatchBytes() = 64 << 10;  // about 20 batches
        std::vector<Row> rows = Take(FromString(orders)).LeftJoin(cust, {"cust_id"}).LeftJoin(prod).ToRows();
        CHECK(rows.size() == (size_t)nord);
        int unknown_cust = 0, unknown_prod = 0, both = 0;
        for (int i = 0; i < nord; i++) {
            const Row& r = rows[i];
            auto c = name.find(ord[i][1]);
            auto p = price.find(ord[i][2]);
            CHECK(r.at("order_id") == ord[i][0] && r.at("cust_id") == ord[i][1] && r.at("prod_id") == ord[i][2]);
            CHECK(r.at("id") == (c != name.end() ? ord[i][1] : std::string()));  // the index key named unlike cust_id
            CHECK(r.at("name") == (c != name.end() ? c->second : std::string()));
            CHECK(r.at("price") == (p != price.end() ? p->second : std::string()));
            unknown_cust += c == name.end();
            unknown_prod += p == price.end();
            both += c != name.end() && p != price.end();
            if (i < 40 && (c == name.end() || p == price.end()))
                printf("order %s: %s%s\n", ord[i][0].c_str(), c == name.end() ? "unknown customer " : "", p == price.end() ? "unknown product" : "");
        }
        // the matched rows are Join's result
        std::vector<Row> inner = Take(FromString(orders)).Join(cust, {"cust_id"}).Join(prod).ToRows();
        CHECK(inner.size() == (size_t)both);
        size_t k = 0;
        for (const Row& r : rows)
            if (!r.at("id").empty() && !r.at("price").empty()) { CHECK(k < inner.size() && r == inner[k]); k++; }
        CHECK(k == inner.size());
        bool threw = false;
        try { Take(FromString(orders)).LeftJoin(cust, {"a", "b"}); } catch (const std::logic_error& e) { threw = std::string(e.what()) == "too many source columns in LeftJoin()"; }
        CHECK(threw);
        printf("%d orders: %d with an unknown customer, %d with an unknown product\n", nord, unknown_cust, unknown_prod);
        CHECK(unknown_cust > 0 && unknown_prod > 0);
        printf("left join example ok\n");
    } catch (const std::exception& e) {
        fprintf(stderr, "error: %s\n", e.what());
        return 1;
    }
    return 0;
}
