// example.cpp — the reference's README / test scenarios through the C++ host mirror (host/csvplus.hpp).
// Mirrors TestSimpleDataSource (csvplus_test.go:118-151), TestSimpleUniqueJoin (:368-452), TestErrors (:808-909),
// TestWriteFile (:172-196), TestJSONStruct (:1016-1048) and TestSimpleTotals (:516-571) on fixtures generated like
// csvplus_test.go:1207-1333.
// Exit code 0 = all checks hold.
#include <unistd.h>

#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <cstring>
#include <sstream>

#include "csvplus.hpp"

using namespace csvplus;

#define CHECK(c) do { if (!(c)) { fprintf(stderr, "CHECK failed %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

int main() {
    const char* names[] = {"Amelia", "Olivia", "Emily", "Ava", "Isla", "Oliver", "Jack", "Harry", "Jacob", "Charlie"};
    const char* surnames[] = {"Smith", "Jones", "Taylor", "Williams", "Brown", "Davies", "Evans", "Wilson", "Thomas", "Roberts", "Johnson", "Lewis"};
    std::string people = "id,name,surname,born\n";
    for (int i = 0; i < 10; i++) for (int j = 0; j < 12; j++)
        people += std::to_string(i * 12 + j) + "," + names[i] + "," + surnames[j] + "," + std::to_string(1916 + (i * 37 + j * 11) % 90) + "\n";
    std::string orders = "order_id,cust_id,prod_id,qty,ts\n";
    std::vector<int> cust(10000), qty(10000);
    unsigned s = 12345;
    for (int i = 0; i < 10000; i++) {
        s = s * 1103515245u + 12345u; cust[i] = (s >> 8) % 120;
        s = s * 1103515245u + 12345u; qty[i] = 1 + (s >> 8) % 100;
        orders += std::to_string(i) + "," + std::to_string(cust[i]) + "," + std::to_string(i % 8) + "," + std::to_string(qty[i]) + ",2016-09-14T08:48:22+01:00\n";
    }
    try {
        // TestSimpleDataSource
        auto src = Take(FromString(people).SelectColumns({"born", "id", "name", "surname"}))
                       .Filter(Any({Like({{"name", "Jack"}}), Like({{"name", "Amelia"}})}));
        int n = 0;
        src([&](const Row& row) { if ((row.at("name") == "Jack" || row.at("name") == "Amelia") && row.size() == 4) n++; });
        CHECK(n == 24);
        // TestSimpleUniqueJoin
        auto idx = Take(FromString(people).SelectColumns({"id", "name", "surname"})).UniqueIndexOn({"id"});
        std::vector<long> qsum(120, 0), want(120, 0);
        for (int i = 0; i < 10000; i++) want[cust[i]] += qty[i];
        long joined = 0;
        Take(FromString(orders).SelectColumns({"order_id", "cust_id", "qty"})).Join(idx, {"cust_id"})([&](const Row& row) {
            if (row.size() == 6 && row.at("id") == row.at("cust_id")) { qsum[std::stoi(row.at("id"))] += std::stol(row.at("qty")); joined++; }
        });
        CHECK(joined == 10000);
        CHECK(qsum == want);
        // TestWriteFile: parse -> ToCsv round trip
        std::ostringstream out;
        Take(FromString(people).SelectColumns({"id", "name", "surname", "born"})).ToCsv(out, {"id", "name", "surname", "born"});
        CHECK(out.str() == people);
        // TestWriteFile streamed: FromFile -> ToCsvFile with the input parsed in batches of 64 bytes (a few records each)
        {
            char in_name[] = "/tmp/csvplus_example_XXXXXX";
            const int fd = mkstemp(in_name);
            CHECK(fd >= 0);
            CHECK(write(fd, people.data(), people.size()) == (ssize_t)people.size());
            close(fd);
            const std::string out_name = std::string(in_name) + ".out";
            const uint64_t saved = StreamBatchBytes();
            StreamBatchBytes() = 64;
            Take(FromFile(in_name).SelectColumns({"id", "name", "surname", "born"})).ToCsvFile(out_name, {"id", "name", "surname", "born"});
            std::ifstream back(out_name, std::ios::binary);
            std::stringstream got; got << back.rdbuf();
            CHECK(got.str() == people);
            // a join over batches, and a source error in a later batch: the file is removed
            std::ostringstream streamed_js;
            Take(FromString(orders).SelectColumns({"order_id", "cust_id", "qty"})).Join(idx, {"cust_id"}).Top(3).ToJSON(streamed_js);
            long sjoined = 0;
            Take(FromString(orders).SelectColumns({"order_id", "cust_id", "qty"})).Join(idx, {"cust_id"})([&](const Row&) { sjoined++; });
            CHECK(sjoined == 10000);
            try {
                Take(FromString(people + "1,2\n")).ToCsvFile(out_name, {"id"});
                CHECK(false);
            } catch (const DataSourceError& e) { CHECK(std::string(e.what()) == "row 122: wrong number of fields"); }
            std::ifstream gone(out_name);
            CHECK(!gone.good());
            // ToJSON with the error in the first batch of an input pushed in two pieces: the 5 rows before it are written
            // without ']'; pushed in one piece, nothing is written
            size_t at = 0;
            for (int k = 0; k < 6; k++) at = people.find('\n', at) + 1;
            const std::string bad = people.substr(0, at) + "1,2\n" + people.substr(at);
            std::ostringstream top5;
            Take(FromString(people)).Top(5).ToJSON(top5);
            for (uint64_t batch : {(uint64_t)bad.size() / 2 + 1, (uint64_t)bad.size() + 1}) {
                StreamBatchBytes() = batch;
                std::ostringstream js_err;
                try {
                    Take(FromString(bad)).ToJSON(js_err);
                    CHECK(false);
                } catch (const DataSourceError& e) { CHECK(std::string(e.what()) == "row 7: wrong number of fields"); }
                const std::string want = batch <= bad.size() ? top5.str().substr(0, top5.str().size() - 1) : "";
                CHECK(js_err.str() == want);
            }
            StreamBatchBytes() = saved;
            std::ostringstream whole_js;
            Take(FromString(orders).SelectColumns({"order_id", "cust_id", "qty"})).Join(idx, {"cust_id"}).Top(3).ToJSON(whole_js);
            CHECK(streamed_js.str() == whole_js.str() && whole_js.str().size() > 100);
            std::remove(in_name);
        }
        // TestJSONStruct (csvplus_test.go:1016): SelectColumns -> ToJSON, keys sorted, one object per line
        std::ostringstream js, want_js;
        Take(FromString(people).SelectColumns({"name", "surname", "born"})).ToJSON(js);
        want_js << '[';
        for (int i = 0; i < 10; i++) for (int j = 0; j < 12; j++)
            want_js << (i || j ? "," : "") << "{\"born\":\"" << 1916 + (i * 37 + j * 11) % 90 << "\",\"name\":\"" << names[i]
                    << "\",\"surname\":\"" << surnames[j] << "\"}\n";
        want_js << ']';
        CHECK(js.str() == want_js.str());
        // TestSimpleTotals (csvplus_test.go:516): orders x products, cust_id / qty / price converted on the GPU
        std::string stock = "prod_id,product,price\n";
        const double prices[8] = {1.25, 10.5, 3.75, 99.99, 0.5, 12.5, 7.3, 100.01};
        for (int i = 0; i < 8; i++) { char b[64]; snprintf(b, sizeof b, "%d,item%d,%g\n", i, i, prices[i]); stock += b; }
        auto prod = Take(FromString(stock).SelectColumns({"prod_id", "price"})).UniqueIndexOn({"prod_id"});
        Table jt = Take(FromString(orders).SelectColumns({"cust_id", "prod_id", "qty"})).Join(prod).ToTable();
        const int64_t jn = jt.size();
        CHECK(jn == 10000);
        void *d_id = nullptr, *d_qty = nullptr, *d_price = nullptr;
        CHECK(cpb_device_alloc(detail::ctx(), jn * 8, &d_id) == CPB_OK && cpb_device_alloc(detail::ctx(), jn * 8, &d_qty) == CPB_OK &&
              cpb_device_alloc(detail::ctx(), jn * 8, &d_price) == CPB_OK);
        CHECK(jt.ValuesAsInt("cust_id", (int64_t*)d_id) == 0);
        CHECK(jt.ValuesAsInt("qty", (int64_t*)d_qty) == 0);
        CHECK(jt.ValuesAsFloat64("price", (double*)d_price) == 0);
        std::vector<int64_t> hid(jn), hqty(jn); std::vector<double> hprice(jn);
        CHECK(cpb_memcpy_d2h(detail::ctx(), hid.data(), d_id, jn * 8) == CPB_OK && cpb_memcpy_d2h(detail::ctx(), hqty.data(), d_qty, jn * 8) == CPB_OK &&
              cpb_memcpy_d2h(detail::ctx(), hprice.data(), d_price, jn * 8) == CPB_OK);
        std::vector<double> totals(120, 0), want_totals(120, 0);
        for (int64_t i = 0; i < jn; i++) { CHECK(hid[i] >= 0 && hid[i] < 120); totals[hid[i]] = hprice[i] * (double)hqty[i]; }
        for (int i = 0; i < 10000; i++) want_totals[cust[i]] = prices[i % 8] * (double)qty[i];
        CHECK(totals == want_totals);
        // a failing row: the reference's text, strict and not
        try { jt.ValuesAsInt("price", (int64_t*)d_id); CHECK(false); }
        catch (const Error& e) { CHECK(std::string(e.what()).find("column \"price\": cannot convert \"") == 0 &&
                                       std::string(e.what()).find("\" to integer: invalid syntax") != std::string::npos); }
        CHECK(jt.ValuesAsInt("price", (int64_t*)d_id, nullptr, false) == 10000);
        try { jt.ValuesAsFloat64("xxx", (double*)d_price); CHECK(false); }
        catch (const Error& e) { CHECK(std::string(e.what()) == "missing column \"xxx\""); }
        cpb_device_free(detail::ctx(), d_id); cpb_device_free(detail::ctx(), d_qty); cpb_device_free(detail::ctx(), d_price);
        // TestErrors
        try { Take(FromString(people).SelectColumns({"id", "name", "xxx"})).ToRows(); CHECK(false); }
        catch (const DataSourceError& e) { CHECK(std::string(e.what()) == "row 1: column not found: xxx"); }
        try { Take(FromString(people).SelectColumns({"id", "name", "surname"})).UniqueIndexOn({"name"}); CHECK(false); }
        catch (const Error& e) { CHECK(std::string(e.what()).find("duplicate value while creating unique index: { \"name\" : \"Amelia\" }") == 0); }
        try { Take(FromString(people).SelectColumns({"id", "name"})).IndexOn({"name", "xxx"}); CHECK(false); }
        catch (const DataSourceError& e) { CHECK(std::string(e.what()).find("missing column \"xxx\" while creating an index") != std::string::npos); }
        // ResolveDuplicates + Find (TestErrors :845-863, TestIndexImpl)
        auto byname = Take(FromString(people).SelectColumns({"id", "name", "surname"})).IndexOn({"name"});
        byname.ResolveDuplicates([](const std::vector<Row>& g) { return g.size() == 12 ? 0L : -1L; });
        CHECK(byname.size() == 10);
        CHECK(byname.Find({"Jack"}).ToRows().size() == 1);
        // host closure boundary: Filter(func) + Map then a device join again
        auto rows = Take(FromString(orders)).Filter(Func([](const Row& r) { return std::stoi(r.at("qty")) > 90; }))
                        .Map([](const Row& r) { Row x = r; x["tag"] = "big"; return x; }).Join(idx, {"cust_id"}).Top(5).ToRows();
        CHECK(rows.size() == 5 && rows[0].at("tag") == "big" && rows[0].count("surname") == 1);
    } catch (const std::exception& e) {
        fprintf(stderr, "exception: %s\n", e.what());
        return 2;
    }
    // ---- multi-GPU entry points of the C ABI (SURVEY §8e), on as many devices as the box has (at most 2 here): the build
    // side is parsed in row-range shards, one per context, all-gathered (cpb_allgather_tables) and indexed on every rank;
    // every rank joins its own probe shard; the concatenation of the results equals the single-GPU join.
    {
        int ndev = 0;
        for (int d = 0; d < 2; d++) { cpb_ctx* probe = nullptr; if (cpb_init(d, &probe) == CPB_OK) { ndev++; cpb_shutdown(probe); } else break; }
        CHECK(ndev >= 1);
        std::vector<int> devs(ndev);
        for (int d = 0; d < ndev; d++) devs[d] = d;
        std::vector<cpb_ctx*> cs(ndev, nullptr);
        CHECK(cpb_init_multi(devs.data(), ndev, cs.data()) == CPB_OK);
        CHECK(cpb_comm_size(cs[0]) == ndev && cpb_comm_rank(cs[ndev - 1]) == ndev - 1);
        auto cs_ = [](const char* s) { return cpb_str{s, strlen(s)}; };
        cpb_reader_opts opts{',', 0, 0, 0, 0, 1, 0};
        cpb_header_col cust_spec[3] = {{cs_("id"), -1, 0}, {cs_("name"), -1, 0}, {cs_("surname"), -1, 0}};
        // row-range shards of the people file: the header + a contiguous run of lines per rank
        std::vector<std::string> lines;
        { std::istringstream in(people); std::string ln; while (std::getline(in, ln)) lines.push_back(ln + "\n"); }
        std::vector<cpb_table*> locals(ndev, nullptr), gathered(ndev, nullptr);
        cpb_error e;
        for (int r = 0; r < ndev; r++) {
            std::string shard = lines[0];
            const size_t lo = 1 + (lines.size() - 1) * r / ndev, hi = 1 + (lines.size() - 1) * (r + 1) / ndev;
            for (size_t i = lo; i < hi; i++) shard += lines[i];
            CHECK(cpb_parse_csv(cs[r], shard.data(), shard.size(), 0, &opts, cust_spec, 3, nullptr, &locals[r], &e) == CPB_OK);
        }
        CHECK(cpb_allgather_tables(cs.data(), locals.data(), ndev, gathered.data()) == CPB_OK);
        long total = 0;
        for (int r = 0; r < ndev; r++) {
            CHECK(cpb_table_num_rows(gathered[r]) == 120);
            cpb_index* ix = nullptr;
            cpb_str key = cs_("id");
            CHECK(cpb_index_build(cs[r], gathered[r], &key, 1, 1, &ix, &e) == CPB_OK);
            // this rank's probe shard: a row range of the orders file
            std::vector<std::string> ol;
            { std::istringstream in(orders); std::string ln; while (std::getline(in, ln)) ol.push_back(ln + "\n"); }
            std::string shard = ol[0];
            const size_t lo = 1 + (ol.size() - 1) * r / ndev, hi = 1 + (ol.size() - 1) * (r + 1) / ndev;
            for (size_t i = lo; i < hi; i++) shard += ol[i];
            cpb_header_col ord_spec[2] = {{cs_("cust_id"), -1, 0}, {cs_("qty"), -1, 0}};
            cpb_table *probe = nullptr, *joined = nullptr;
            CHECK(cpb_parse_csv(cs[r], shard.data(), shard.size(), 0, &opts, ord_spec, 2, nullptr, &probe, &e) == CPB_OK);
            cpb_str jc = cs_("cust_id");
            CHECK(cpb_join(cs[r], probe, ix, &jc, 1, &joined, &e) == CPB_OK);
            CHECK(cpb_table_num_rows(joined) == (int64_t)(hi - lo) && cpb_table_num_cols(joined) == 5);
            total += (long)cpb_table_num_rows(joined);
            cpb_table_free(joined); cpb_table_free(probe); cpb_index_free(ix);
        }
        CHECK(total == 10000);
        // the metadata exchange of byte-range shards
        uint64_t in2[2] = {7, 9}, out2[2 * 2] = {0, 0, 0, 0};
        if (ndev == 1) { CHECK(cpb_allgather_u64(cs[0], in2, 2, out2) == CPB_OK && out2[0] == 7 && out2[1] == 9); }
        for (int r = 0; r < ndev; r++) { cpb_table_free(gathered[r]); cpb_table_free(locals[r]); }
        for (int r = 0; r < ndev; r++) cpb_shutdown(cs[r]);
        printf("multi-GPU entry points ok on %d device(s)\n", ndev);
    }
    printf("host example ok\n");
    return 0;
}
