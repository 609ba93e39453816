"""Host-side helpers of bench.py that must not depend on a GPU: the NUMA binding (best effort, never raises), the
workload description, the duplicate resolver and the output dump."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def test_numa_binding_is_best_effort():
    before = os.sched_getaffinity(0)
    assert bench.bind_to_gpu_numa_node(0) is None or isinstance(bench.bind_to_gpu_numa_node(0), int)
    assert os.sched_getaffinity(0) <= before  # never widens, never raises without a GPU


def test_workload_config_names_the_baseline_configs():
    cfg = bench.workload_config(1)
    assert "workload" in cfg and "model" not in cfg and cfg["orders_rows_per_gpu"] == 125_000_000
    assert cfg["customers_rows"] == 100_000_000 and cfg["products_rows"] == 1_000_000  # BASELINE configs[3] at --gpus 8
    assert "NCCL" in bench.workload_config(4)["parallelism"]
    ref = bench.workload_config(1, ref=(2_000_000, 1_600_000, 100_000))  # the reference arm states the sample it ran
    assert ref["orders_rows_per_gpu"] == 2_000_000 and ref["customers_rows"] == 1_600_000


def test_min_id_resolver_keeps_bytewise_smallest():
    import numpy as np

    class FakeTable:
        def __init__(self, vals):
            self.vals = vals

        def column(self, name):
            off = np.zeros(len(self.vals) + 1, np.int64); off[1:] = np.cumsum([len(v) for v in self.vals])
            return off, np.frombuffer(b"".join(self.vals), np.uint8)
    vals = [b"7", b"10", b"9", b"100", b"3", b"21", b"2", b"20", b"5"]
    lo, hi = np.array([1, 5], np.int64), np.array([4, 8], np.int64)  # groups [1,4) and [5,8)
    keep = bench.min_id_resolver(FakeTable(vals), lo, hi)
    # bytewise: "10" < "100" < "9" ; "2" < "20" < "21"
    assert keep.tolist() == [1, 6]
    assert bench.index_sides(10_000_000) == 3794


def test_dump_table_writes_a_fixed_float_sample(tmp_path):
    import numpy as np

    class FakeTable:
        columns = ["k", "v"]

        def __init__(self, n):
            self.vals = {"k": [b"%d" % i for i in range(n)], "v": [b"x" * (i % 5) for i in range(n)]}

        def __len__(self):
            return len(self.vals["k"])

        def column(self, name, lo, hi):
            vals = self.vals[name][lo:hi]
            off = np.zeros(len(vals) + 1, np.int64); off[1:] = np.cumsum([len(v) for v in vals])
            return off, np.frombuffer(b"".join(vals), np.uint8)
    for run in ("a", "b"):
        bench.dump_table(str(tmp_path / run), "t", FakeTable(10_000))
    files = sorted(p.name for p in (tmp_path / "a").iterdir())
    assert files == ["t.k_bytes.npy", "t.k_len.npy", "t.v_bytes.npy", "t.v_len.npy", "t_num_rows.npy", "t_rows.npy"]
    for f in files:
        x, y = np.load(tmp_path / "a" / f), np.load(tmp_path / "b" / f)
        assert x.dtype in (np.float32, np.float64) and np.array_equal(x, y)
    rows = np.load(tmp_path / "a" / "t_rows.npy").astype(np.int64)
    assert len(rows) == bench.DUMP_BLOCKS * bench.DUMP_BLOCK_ROWS and rows.max() < 10_000
    k = np.load(tmp_path / "a" / "t.k_bytes.npy"); kl = np.load(tmp_path / "a" / "t.k_len.npy").astype(np.int64)
    for i in (0, 777, len(rows) - 1):
        assert bytes(k[i, :kl[i]].astype(np.uint8)) == b"%d" % rows[i]
    bench.dump_table(str(tmp_path / "small"), "t", FakeTable(3))
    assert np.load(tmp_path / "small" / "t_rows.npy").tolist() == [0, 1, 2]
