"""Host-side checks of the CSV scan's yardsticks (no GPU): the reference reader of csv_reference.py is pinned against the
hand-written expectations of the edge-shape files, the exact float rounding against known bit patterns, and the .tbl
schema / writer against the reference's TPC-H fixtures."""
import os
from fractions import Fraction

import pytest

import csv_reference as R
import test_gpu_csv_scan as T
from ballista_b200 import tpch

CSV_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "csv")

# pyarrow's rules differ from the scan's for these shapes (a leading '+' on integers, booleans spelled in mixed case,
# empty files); they are checked against the hand-written expectations only
PYARROW_DIFFERS = {"ints", "bools", "empty", "header_only", "decimals"}


@pytest.mark.parametrize("name,data,schema,opts", [e for e in T.EDGE if e[0] not in PYARROW_DIFFERS],
                         ids=[e[0] for e in T.EDGE if e[0] not in PYARROW_DIFFERS])
def test_reference_reader_matches_hand_written_rows(tmp_path, name, data, schema, opts):
    path = T.write(tmp_path, data)
    kw = {k: v for k, v in opts.items() if k in ("delimiter", "quote", "escape", "has_header")}
    got = R.read(path, schema, **kw)
    assert {n: R.canon_values(got.column(n)) for n in got.column_names} == R.expected_edge(name)


def test_f32_rounding_is_exact():
    assert R.f32_bits("16777217") == 0x4B800000          # halfway between 2^24 and 2^24 + 2: to even
    assert R.f32_bits("16777219") == 0x4B800002          # halfway: to even (up)
    assert R.f32_bits("1.40129846e-45") == 1             # smallest subnormal
    assert R.f32_bits("7.0064924e-46") == 1              # just above half of it
    assert R.f32_bits("7.00649232e-46") == 0             # just below
    assert R.f32_bits(R.fraction_to_decimal(Fraction(1, 2 ** 150))) == 0   # exactly half: to even (zero)
    assert R.f32_bits(str(2 ** 128 - 2 ** 103)) == 0x7F800000     # halfway to 2^128: to even (infinity)
    assert R.f32_bits("3.4028235677973366e38") == 0x7F7FFFFF     # just below it
    assert R.f32_bits("-0") == 0x80000000 and R.f32_bits("-inf") == 0xFF800000
    # a double rounding would get this one wrong: the decimal lies just above a float halfway point, its double below it
    s = R.fraction_to_decimal(Fraction(2 ** 24 + 1, 2 ** 24) + Fraction(1, 2 ** 80))
    assert R.f32_bits(s) == 0x3F800001 and R.b32(float(s)) == 0x3F800000


def test_tbl_schema_and_writer(oracle, oracle_lib, tmp_path):
    sch = tpch.tbl_schema("lineitem")
    assert [f["name"] for f in sch][-1] == "__placeholder" and len(sch) == 17
    for name in ("nation", "lineitem_partition0"):
        table = name.split("_")[0]
        t = R.read(os.path.join(CSV_DIR, name + ".tbl"), tpch.tbl_schema(table), delimiter="|")
        assert t.num_rows > 0 and t.column("__placeholder").null_count == t.num_rows
    host, path = T._lineitem_tbl(oracle, oracle_lib, tmp_path, msf=1)
    back = R.read(path, sch, delimiter="|")
    assert back.num_rows == host.num_rows
    for n in host.column_names:
        assert back.column(n).to_pylist() == host.column(n).to_pylist(), n
    with open(path, "rb") as f:
        assert f.readline().endswith(b"|\n")
