// sprintf_example.cpp — the README's second example through the C++ mirror (host/csvplus.hpp): orders joined with their
// customers and products, every joined row printed by the RowFunc's fmt.Printf line, here formatted on the GPU
// (DataSource::ToText) and written to stdout.  Then one computed column (Table::WithSprintf) and a refused format.
//   sprintf_example <people.csv> <orders.csv>
#include <iostream>

#include "csvplus.hpp"

using namespace csvplus;

int main(int argc, char** argv) {
    if (argc != 3) { std::cerr << "usage: sprintf_example <people.csv> <orders.csv>\n"; return 2; }
    const char* names[] = {"apple", "pear", "plum", "fig", "lime", "kiwi", "date", "quince"};
    std::string products = "prod_id,product,price\n";
    for (int i = 0; i < 8; i++) products += std::to_string(i) + "," + names[i] + "," + std::to_string(i * 3 + 1) + "." + std::to_string(10 + i * 7) + "\n";
    Index cust = Take(FromFile(argv[1]).SelectColumns({"id", "name", "surname"})).UniqueIndexOn({"id"});
    Index prod = Take(FromString(products)).UniqueIndexOn({"prod_id"});
    DataSource joined = Take(FromFile(argv[2]).SelectColumns({"cust_id", "prod_id", "qty", "ts"})).Join(cust, {"cust_id"}).Join(prod);
    joined.ToText(std::cout, "%s %s bought %s %ss for \xc2\xa3%s each on %s\n", {"name", "surname", "qty", "product", "price", "ts"});
    Table t = joined.Top(3).ToTable().WithSprintf("label", "%-8s|%.3s|%5v", {"name", "surname", "qty"});
    for (const Row& r : t.rows()) std::cout << "label " << r.at("label") << "\n";
    try {
        t.WithSprintf("bad", "%d", {"qty"});
        std::cout << "no error\n";
    } catch (const Error& e) {
        std::cout << "error: " << e.what() << "\n";
    }
    return 0;
}
