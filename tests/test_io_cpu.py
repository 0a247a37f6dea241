"""CPU tests of the reference's text formats (fplll_b200/io.py, SURVEY §8 f3): matrices written by the reference's own
latticegen / read back by its own reader (stored under tests/golden), strategies/default.json against the committed
array form, the GSO dump record."""
import json
import os

import numpy as np
import pytest

from fplll_b200 import io as fio
import helpers as H

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")


def test_matrix_text_format_round_trips_through_the_reference(tmp_path):
    # written by the reference's own latticegen (Matrix<T>::print): `latticegen r 12 200`, 12 x 13, 200-bit entries
    txt = open(os.path.join(GOLD, "latticegen_r_12_200.txt")).read()
    a = fio.read_matrix(txt)
    assert a.shape == (12, 13) and int(a[0, 0]).bit_length() > 64
    p = str(tmp_path / "m.txt")
    fio.write_matrix(p, a)
    # the reference's own reader accepted our output and printed it back identically (ref_probe's load/save pair:
    # Matrix<T>::read then print, tests/golden/make_golden.py --live)
    q = os.path.join(GOLD, "latticegen_r_12_200_resaved.txt")
    assert np.array_equal(fio.read_matrix(q), a)
    assert open(q).read().split() == open(p).read().split() == fio.write_matrix(None, a).split()


def test_read_matrix_pads_short_rows_and_refuses_overflow():
    a = fio.read_matrix("[[1 2 3]\n[4]\n[5 6]]")
    assert a.tolist() == [[1, 2, 3], [4, 0, 0], [5, 6, 0]]
    with pytest.raises(OverflowError):
        fio.read_matrix("[[%d]]" % (1 << 70), dtype=np.int64)


def test_strategies_json_equals_the_committed_table():
    """the committed table (fplll_b200/data) is the reference's strategies/default.json: every block size's arrays hash
    like the reference file's parsed with load_strategies_json, and the parser reads an excerpt of that file."""
    from fplll_b200.bkz import load_strategies
    want = load_strategies()
    digests = json.load(open(os.path.join(GOLD, "strategies_default_digests.json")))
    assert sorted(int(bs) for bs in digests) == sorted(want)
    for bs in want:
        assert H.strategy_digest(want[bs]) == digests[str(bs)], bs
    got = fio.load_strategies_json(os.path.join(GOLD, "strategies_default_excerpt.json"))
    assert sorted(got) == [0, 1, 2, 10, 20]
    for bs in got:
        for x, y in zip(got[bs], want[bs]):
            assert np.array_equal(np.asarray(x), np.asarray(y)), bs


def test_gso_dump_is_the_reference_json_shape(tmp_path):
    p = str(tmp_path / "dump.json")
    d = fio.GSODump(p)
    d.append("Input", -1, 0.0, [0.75, 0.5], [10, 8])
    d.append("Output", 3, 1.5, [0.75, 0.5], [9, 8])
    recs = json.load(open(p))
    assert [r["step"] for r in recs] == ["Input", "Output"] and recs[1]["loop"] == 3
    assert abs(recs[0]["norms"][0] - (np.log(0.75) + 10 * np.log(2.0))) < 1e-6
