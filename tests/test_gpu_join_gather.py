"""GPU parity of the index-row gather of Join: index key columns taken from the probe, row slots, the staged slot copy.
Every result is compared with the CPU oracle's mergeRows (csvplus.go:571-583) byte for byte."""
import random

import pytest

from oracle import oracle as orc
from tests.helpers import assert_table_equals_oracle, gpu_ctx

pytestmark = pytest.mark.gpu


def _csv(header, rows):
    return (",".join(header) + "\n" + "".join(",".join(r) + "\n" for r in rows)).encode()


def _word(rng, lo, hi):
    return "".join(rng.choice("abcxyz01") for _ in range(rng.randrange(lo, hi + 1)))


def test_join_probe_key_column_is_a_row_range_view():
    """the index key column of the result is the probe's key column: also when that column is a row-range view"""
    import csvplus_b200 as cp
    rng = random.Random(11)
    nidx = 3000
    idata = _csv(["id", "name", "surname"], [[str(i), _word(rng, 1, 7), _word(rng, 1, 8)] for i in range(nidx)])
    pdata = _csv(["cust_id", "qty"], [[str(rng.randrange(nidx)), str(j)] for j in range(9000)])
    ctx = gpu_ctx()
    ti, _ = cp.parse_csv(ctx, idata)
    tp, _ = cp.parse_csv(ctx, pdata)
    idx = ti.index_on("id", unique=True)
    oidx = orc.reader_rows(idata).unique_index_on("id")
    for lo, hi in ((1234, 8000), (4321, 4322), (0, 9000)):
        view = tp.slice(lo, hi)
        assert_table_equals_oracle(view.join(idx, "cust_id"), orc.reader_rows(pdata).drop(lo).top(hi - lo).join(oidx, "cust_id"))


def test_join_prefix_of_composite_index_shares_only_the_first_key_column():
    """a join on the first of two key columns: k1 comes from the probe, k2 (a key column not joined on) is gathered"""
    import csvplus_b200 as cp
    rng = random.Random(12)
    irows = [[str(rng.randrange(400)), _word(rng, 0, 6), _word(rng, 0, 9)] for _ in range(2000)]
    idata = _csv(["k1", "k2", "v"], irows)
    pdata = _csv(["a", "p"], [[str(rng.randrange(420)), str(j)] for j in range(5000)])
    ctx = gpu_ctx()
    ti, _ = cp.parse_csv(ctx, idata)
    tp, _ = cp.parse_csv(ctx, pdata)
    idx = ti.index_on("k1", "k2")
    oidx = orc.reader_rows(idata).index_on("k1", "k2")
    j = tp.join(idx, "a")
    assert j.columns == ["k1", "k2", "v", "a", "p"]
    oj = orc.reader_rows(pdata).join(oidx, "a")
    assert len(oj) > 5000
    assert_table_equals_oracle(j, oj)
    # both key columns joined: k1 and k2 both come from the probe, only v is gathered
    pdata2 = _csv(["x", "y"], [irows[rng.randrange(len(irows))][:2] for _ in range(3000)])
    tp2, _ = cp.parse_csv(ctx, pdata2)
    assert_table_equals_oracle(tp2.join(idx, "x", "y"), orc.reader_rows(pdata2).join(oidx, "x", "y"))


def test_unique_join_with_a_few_missing_keys_at_scale():
    """a unique-index join where a few probe keys have no match: not every probe row matches once, so the result is
    built from (probe row, index row) pairs, with the index key column gathered from the probe side"""
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    ncust, nord = 200_000, 400_000
    cust = ctx.gen_csv("customers", (0, ncust), n_cust=ncust, permute=True)
    orders = ctx.gen_csv("orders", (0, nord), n_cust=ncust + 7, n_prod=100)  # ids >= ncust have no customer
    spec_c = [("id", -1), ("name", -1), ("surname", -1)]
    spec_o = [("cust_id", -1), ("prod_id", -1), ("qty", -1), ("ts", -1)]
    tc, _ = cp.parse_csv(ctx, cust, spec=spec_c)
    to, _ = cp.parse_csv(ctx, orders, spec=spec_o)
    j = to.join(tc.index_on("id", unique=True), "cust_id")
    oc = orc.reader_rows(cust.to_host(), select=[c for c, _ in spec_c])
    oj = orc.reader_rows(orders.to_host(), select=[c for c, _ in spec_o]).join(oc.unique_index_on("id"), "cust_id")
    assert 0 < nord - len(oj) < nord // 1000
    assert_table_equals_oracle(j, oj)


@pytest.mark.parametrize("shape", ["one_column", "two_columns"])
def test_slot_copy_group_straddling_the_stage(shape):
    """64-byte row slots: a warp's 32 rows then carry up to 2 KiB of one column, and a group whose bytes do not fit
    the staging buffer (from its 16-byte aligned start) is copied straight to the destination instead"""
    import csvplus_b200 as cp
    rng = random.Random(13)
    nidx = 5000

    def val(i, n):
        return "".join(rng.choice("abcdefgh") for _ in range(n - (1 if i % 37 == 5 else 0)))
    if shape == "one_column":
        hdr, mk = ["k", "a"], (lambda i: [str(i), val(i, 64)])
    else:
        hdr, mk = ["k", "a", "b"], (lambda i: [str(i), val(i, 32), val(i + 1, 32)])
    idata = _csv(hdr, [mk(i) for i in range(nidx)])
    pdata = _csv(["k2"], [[str(rng.randrange(nidx))] for _ in range(12000)])
    ctx = gpu_ctx()
    ti, _ = cp.parse_csv(ctx, idata)
    tp, _ = cp.parse_csv(ctx, pdata)
    oidx = orc.reader_rows(idata).unique_index_on("k")
    assert_table_equals_oracle(tp.join(ti.index_on("k", unique=True), "k2"), orc.reader_rows(pdata).join(oidx, "k2"))
    # a non-unique index takes the row slots over the sorted order
    assert_table_equals_oracle(tp.join(ti.index_on("k"), "k2"), orc.reader_rows(pdata).join(orc.reader_rows(idata).index_on("k"), "k2"))
