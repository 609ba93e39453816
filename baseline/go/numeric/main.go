// Regenerates tests/golden/numeric_kat.expected with Go's own strconv (the functions behind the reference's
// Row.ValueAsInt / Row.ValueAsFloat64, csvplus.go:163-205):
//
//	go run ./numeric ../../tests/golden/numeric_kat.csv > /tmp/numeric_kat.expected
//	cmp ../../tests/golden/numeric_kat.expected /tmp/numeric_kat.expected
//
// One line per row of the CSV's column `s`: `<Atoi value> <Atoi status> <ParseFloat bits, 16 hex digits> <ParseFloat
// status>`, status 0 ok, 1 ErrSyntax, 2 ErrRange, values being what strconv returns alongside the error.  Go 1.23
// (go.mod of the reference).  Never compiled here (no Go toolchain in this image).
//
// With -32 it regenerates tests/golden/numeric32_kat.expected from numeric32_kat.csv instead: one line per row,
// `<ParseFloat(s, 32) bits, 8 hex digits> <status>`:
//
//	go run ./numeric -32 ../../tests/golden/numeric32_kat.csv > /tmp/numeric32_kat.expected
//	cmp ../../tests/golden/numeric32_kat.expected /tmp/numeric32_kat.expected
package main

import (
	"encoding/csv"
	"errors"
	"fmt"
	"log"
	"math"
	"os"
	"strconv"
)

func status(err error) int {
	switch {
	case err == nil:
		return 0
	case errors.Is(err, strconv.ErrSyntax):
		return 1
	case errors.Is(err, strconv.ErrRange):
		return 2
	}
	log.Fatalf("unexpected error %v", err)
	return -1
}

func main() {
	args := os.Args[1:]
	bits32 := len(args) > 0 && args[0] == "-32"
	if bits32 {
		args = args[1:]
	}
	f, err := os.Open(args[0])
	if err != nil {
		log.Fatal(err)
	}
	defer f.Close()
	records, err := csv.NewReader(f).ReadAll()
	if err != nil {
		log.Fatal(err)
	}
	if len(records) == 0 || len(records[0]) != 1 || records[0][0] != "s" {
		log.Fatal("expected a single column named s")
	}
	for _, rec := range records[1:] {
		if bits32 {
			x, ferr := strconv.ParseFloat(rec[0], 32)
			fmt.Printf("%08x %d\n", math.Float32bits(float32(x)), status(ferr))
			continue
		}
		i, ierr := strconv.Atoi(rec[0])
		x, ferr := strconv.ParseFloat(rec[0], 64)
		fmt.Printf("%d %d %016x %d\n", i, status(ierr), math.Float64bits(x), status(ferr))
	}
}
