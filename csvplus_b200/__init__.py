"""csvplus_b200 — H100-native columnar CSV ETL hot path with the csvplus API names.

Product path = csvplus_b200/libcsvplus_b200.so (hand-written sm_90a CUDA kernels behind the C ABI
of include/csvplus_b200.h).  This package is the thin host mirror of the reference's Go API
(csvplus.go) over that ABI; it never computes results on the CPU and fails loudly when the CUDA
library or a GPU is missing.
"""
from .api import (All, Any, Categories, Context, CsvPlusError, DataSource, DataSourceError, DeviceBuffer, FormatFloat, FromBytes,  # noqa: F401
                  FromFile, FromReadCloser, FromReader, Groups, HostBuffer, Index, Like, LoadIndex, MAX_ORDER_KEYS, Not,
                  ORDER_KINDS, Predicate, Reader, Row, Sprintf,
                  StopIterationEOF, Table, Take, TakeRows, TakeTable, csv_quote_parity, csv_stream_cut, parse_csv, parse_csv_shard)

__all__ = ["All", "Any", "Categories", "Context", "CsvPlusError", "DataSource", "DataSourceError", "DeviceBuffer", "FormatFloat", "FromBytes", "FromFile",
           "FromReadCloser", "FromReader", "Groups", "HostBuffer", "Index", "Like", "LoadIndex", "MAX_ORDER_KEYS", "Not", "ORDER_KINDS", "Predicate", "Reader", "Row",
           "Sprintf", "StopIterationEOF", "Table", "Take", "TakeRows", "TakeTable", "csv_quote_parity", "csv_stream_cut", "parse_csv",
           "parse_csv_shard"]
