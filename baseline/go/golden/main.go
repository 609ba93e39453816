// Regenerates the fixtures of tests/golden/ with the UNMODIFIED reference:
//
//	go run ./golden ../../tests/golden /tmp/golden_from_reference
//	for f in people_amelia orders_join_people orders_without_customer nasty_roundtrip; do
//	    cmp ../../tests/golden/$f.csv /tmp/golden_from_reference/$f.csv; done
//	cmp ../../tests/golden/json_escapes.json /tmp/golden_from_reference/json_escapes.json
//
// Never compiled here (no Go toolchain in this image).  orders_sorted_prod_qty.csv depends on the order of rows
// with equal keys: the reference sorts with sort.Sort (unstable, SURVEY §Q2) while the oracle and the CUDA path keep
// input order, so compare that file after a stable secondary sort on order_id.
package main

import (
	"log"
	"os"
	"path/filepath"

	"github.com/maxim2266/csvplus"
)

func main() {
	in, out := os.Args[1], os.Args[2]
	must := func(err error) {
		if err != nil {
			log.Fatal(err)
		}
	}
	p := func(name string) string { return filepath.Join(in, name) }
	o := func(name string) string { return filepath.Join(out, name) }
	must(os.MkdirAll(out, 0o755))

	// parse + SelectColumns + Filter(Like)
	must(csvplus.Take(csvplus.FromFile(p("people.csv")).SelectColumns("name", "surname", "id")).
		Filter(csvplus.Like(csvplus.Row{"name": "Amelia"})).
		ToCsvFile(o("people_amelia.csv"), "name", "surname", "id"))

	// UniqueIndexOn + Join
	idx, err := csvplus.Take(csvplus.FromFile(p("people.csv")).SelectColumns("id", "name", "surname")).UniqueIndexOn("id")
	must(err)
	must(csvplus.Take(csvplus.FromFile(p("orders.csv")).SelectColumns("order_id", "cust_id", "qty")).
		Join(idx, "cust_id").
		ToCsvFile(o("orders_join_people.csv"), "order_id", "cust_id", "qty", "id", "name", "surname"))

	// IndexOn two columns, iterate in sorted order
	oidx, err := csvplus.Take(csvplus.FromFile(p("orders.csv"))).IndexOn("prod_id", "qty")
	must(err)
	must(csvplus.Take(oidx).ToCsvFile(o("orders_sorted_prod_qty.csv"), "prod_id", "qty", "order_id"))

	// Except
	must(csvplus.Take(csvplus.FromFile(p("orders.csv")).SelectColumns("order_id", "cust_id")).
		Except(idx, "cust_id").
		ToCsvFile(o("orders_without_customer.csv"), "order_id", "cust_id"))

	// reader quoting / CRLF / blank lines -> writer
	must(csvplus.Take(csvplus.FromFile(p("nasty.csv"))).ToCsvFile(o("nasty_roundtrip.csv"), "c0", "c1", "c2", "c3"))

	// every byte class of encoding/json's string encoding, in values and keys (\b and \f since go 1.22)
	must(csvplus.Take(csvplus.FromFile(p("json_escapes.csv"))).ToJSONFile(o("json_escapes.json")))
}
