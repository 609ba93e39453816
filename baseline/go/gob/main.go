// gob/main.go — pins tests/golden/people_index.gob to the reference's own encoding/gob (UNRUN here: no Go toolchain).
//
//	go run ./gob ../../tests/golden
//
// 1. The reference writes IndexOn("id") over SelectColumns("id", "name", "surname") of people.csv (TestIndexStore);
//    its file must decode to the same columns and rows as the golden file (the pair order of its rows is Go's random
//    map order, so the bytes may differ).
// 2. The reference's LoadIndex reads the golden file and iterates the same rows as its own index.
// It also prints the type ids and definition order the reference wrote, which the golden file assumes
// ([]string 65, Row 66, []Row 67; the []Row definition before Row's).
package main

import (
	"bytes"
	"encoding/gob"
	"fmt"
	"os"
	"path/filepath"

	"github.com/maxim2266/csvplus"
)

func rowsOf(ix *csvplus.Index) (out []string) {
	ix.Iterate(func(r csvplus.Row) error { out = append(out, r.String()); return nil })
	return
}

func main() {
	dir := os.Args[1]
	ix, err := csvplus.Take(csvplus.FromFile(filepath.Join(dir, "people.csv")).SelectColumns("id", "name", "surname")).IndexOn("id")
	if err != nil {
		panic(err)
	}
	tmp := filepath.Join(os.TempDir(), "people_index_ref.gob")
	if err = ix.WriteTo(tmp); err != nil {
		panic(err)
	}
	ref, _ := os.ReadFile(tmp)
	golden, _ := os.ReadFile(filepath.Join(dir, "people_index.gob"))
	decode := func(b []byte) (cols []string, rows []map[string]string) {
		dec := gob.NewDecoder(bytes.NewReader(b))
		if err := dec.Decode(&cols); err != nil {
			panic(err)
		}
		if err := dec.Decode(&rows); err != nil {
			panic(err)
		}
		return
	}
	c1, r1 := decode(ref)
	c2, r2 := decode(golden)
	if fmt.Sprint(c1) != fmt.Sprint(c2) || fmt.Sprint(r1) != fmt.Sprint(r2) {
		fmt.Println("MISMATCH: the reference's file and the golden file decode differently")
		os.Exit(1)
	}
	fmt.Printf("reference file: % x ...\n", ref[:64])
	fmt.Printf("golden file:    % x ...\n", golden[:64])
	loaded, err := csvplus.LoadIndex(filepath.Join(dir, "people_index.gob"))
	if err != nil {
		panic(err)
	}
	if fmt.Sprint(rowsOf(loaded)) != fmt.Sprint(rowsOf(ix)) {
		fmt.Println("MISMATCH: LoadIndex(golden) iterates other rows")
		os.Exit(1)
	}
	fmt.Println("gob ok")
}
