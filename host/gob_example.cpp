// gob_example.cpp — Index::WriteTo / LoadIndex of the C++ mirror (host/csvplus.hpp) end to end: the reference's
// TestIndexStore (csvplus_test.go:960-1014) on a people table, plus the error cases of LoadIndex.
#include <unistd.h>

#include <cstdio>
#include <iostream>
#include <iterator>

#include "csvplus.hpp"

using namespace csvplus;

static int fail(const std::string& what) { std::cerr << "FAIL: " << what << "\n"; return 1; }

int main() {
    std::string csv = "id,name,surname,born\n";
    const char* names[] = {"Amelia", "Olivia", "Emily", "Ava", "Isla", "Oliver", "Jack", "Harry", "Jacob", "Charlie"};
    for (int i = 0; i < 300; i++)
        csv += std::to_string((i * 7919) % 300) + "," + names[i % 10] + ",S" + std::to_string(i % 13) + "," + std::to_string(1916 + i % 90) + "\n";
    char dir[] = "/tmp/cpb_gob_XXXXXX";
    if (!mkdtemp(dir)) return fail("mkdtemp");
    const std::string path = std::string(dir) + "/index";

    // TestIndexStore: write, load, compare the key columns and every row
    Index index = Take(FromString(csv).SelectColumns({"id", "name", "surname"})).IndexOn({"id"});
    index.WriteTo(path);
    Index index2 = LoadIndex(path);
    if (index2.columns() != index.columns()) return fail("key columns differ");
    const auto a = Take(index).ToRows(), b = Take(index2).ToRows();
    if (a.size() != b.size() || a.size() != 300) return fail("row count");
    for (size_t i = 0; i < a.size(); i++) if (a[i] != b[i]) return fail("row " + std::to_string(i));
    if (index2.Find({"17"}).ToRows() != index.Find({"17"}).ToRows()) return fail("Find");
    const auto j = TakeRows({{{"id", "42"}, {"x", "1"}}}).Join(index2).ToRows();
    if (j.size() != 1 || j[0].at("name") != index.Find({"42"}).ToRows().at(0).at("name")) return fail("Join");

    // a composite key
    Index ix3 = Take(FromString(csv)).IndexOn({"surname", "name"});
    ix3.WriteTo(path);
    Index ix4 = LoadIndex(path);
    if (ix4.columns() != std::vector<std::string>{"surname", "name"} || Take(ix4).ToRows() != Take(ix3).ToRows()) return fail("composite key");

    // errors: a missing file, an empty file, a cut file; an unwritable path leaves no file
    try { LoadIndex(std::string(dir) + "/missing"); return fail("missing file loaded"); } catch (const Error&) {}
    { std::ofstream(path, std::ios::trunc); }
    try { LoadIndex(path); return fail("empty file loaded"); } catch (const Error& e) { if (std::string(e.what()) != "EOF") return fail(e.what()); }
    index.WriteTo(path);
    {
        std::ifstream f(path, std::ios::binary);
        std::string all((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
        std::ofstream(path, std::ios::binary | std::ios::trunc) << all.substr(0, all.size() - 3);
    }
    try { LoadIndex(path); return fail("cut file loaded"); } catch (const Error& e) { if (std::string(e.what()) != "unexpected EOF") return fail(e.what()); }
    const std::string bad = std::string(dir) + "/no/such/dir/index";
    try { index.WriteTo(bad); return fail("unwritable path written"); } catch (const Error&) {}
    if (access(bad.c_str(), F_OK) == 0) return fail("a file was left behind");

    std::remove(path.c_str());
    rmdir(dir);
    std::cout << "gob example ok\n";
    return 0;
}
