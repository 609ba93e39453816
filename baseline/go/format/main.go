// format regenerates tests/golden/format_kat.csv with Go's strconv and compares it with the committed file, which the
// Python restatement (tests/ftoa_oracle.py) wrote.  Unrun here: there is no Go toolchain in this image.
//
//	go run ./format ../../tests/golden
package main

import (
	"bufio"
	"fmt"
	"math"
	"os"
	"path/filepath"
	"strconv"
	"strings"
)

func main() {
	path := filepath.Join(os.Args[1], "format_kat.csv")
	f, err := os.Open(path)
	if err != nil {
		panic(err)
	}
	defer f.Close()
	bad, n := 0, 0
	sc := bufio.NewScanner(f)
	for sc.Scan() {
		p := strings.SplitN(sc.Text(), ",", 5)
		var got string
		if p[0] == "i" {
			v, err := strconv.ParseInt(p[1], 10, 64)
			if err != nil {
				panic(err)
			}
			got = strconv.FormatInt(v, 10)
		} else {
			u, err := strconv.ParseUint(p[1], 16, 64)
			if err != nil {
				panic(err)
			}
			prec, _ := strconv.Atoi(p[3])
			got = strconv.FormatFloat(math.Float64frombits(u), p[2][0], prec, 64)
		}
		n++
		if got != p[4] {
			bad++
			fmt.Printf("%s %s %s %s: strconv %q, file %q\n", p[0], p[1], p[2], p[3], got, p[4])
		}
	}
	if err := sc.Err(); err != nil {
		panic(err)
	}
	fmt.Printf("%d lines, %d differ\n", n, bad)
	if bad != 0 {
		os.Exit(1)
	}
}
