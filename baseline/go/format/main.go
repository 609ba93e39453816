// format regenerates tests/golden/format_kat.csv and format32_kat.csv with Go's strconv and compares them with the
// committed files, which the Python restatement (tests/ftoa_oracle.py) wrote.  format32_kat.csv lines are
// `bits,fmt,prec,expected` with the float32's bits in hex, checked against FormatFloat(float64(x), fmt, prec, 32).
// Unrun here: there is no Go toolchain in this image.
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
	bad := check(filepath.Join(os.Args[1], "format_kat.csv"), false) + check(filepath.Join(os.Args[1], "format32_kat.csv"), true)
	if bad != 0 {
		os.Exit(1)
	}
}

// check compares one fixture with strconv; bits32: the float32 fixture.  Returns the lines that differ.
func check(path string, bits32 bool) int {
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
		if bits32 {
			p = strings.SplitN(sc.Text(), ",", 4)
			u, err := strconv.ParseUint(p[0], 16, 32)
			if err != nil {
				panic(err)
			}
			prec, _ := strconv.Atoi(p[2])
			got = strconv.FormatFloat(float64(math.Float32frombits(uint32(u))), p[1][0], prec, 32)
			p = append([]string{"f32"}, p...)
		} else if p[0] == "i" {
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
	fmt.Printf("%s: %d lines, %d differ\n", filepath.Base(path), n, bad)
	return bad
}
