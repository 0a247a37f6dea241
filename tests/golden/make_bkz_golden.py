"""Regenerates tests/golden/bkz_driver_ref.npz: what the UNMODIFIED reference's whole bkz_reduction call computes (its
preliminary wrapper LLL, zeros_last / zeros_first, preprocessing, the GH bound, auto-abort, runs to convergence, block
sizes at and above the rank, rank-deficient bases, U), from the reference build in oracle/_ref (oracle/Makefile.ref).
Run in the build container only, after that build:
    python tests/golden/make_bkz_golden.py [OUT.npz]
It compiles bkz_probe.cpp (next to this file) into a temporary directory and runs one probe per case; ~1 min of CPU on
8 cores.  The archive is written with fixed zip timestamps, so that a regeneration is byte-identical.

No case prunes: PruningParams() has expectation 1 (no rerandomisation) and unpruned enumeration returns the shortest
vector of the ball whatever the walk order, so the device driver must end on these bases bit for bit.

Per case <tag>: <tag>_b_in (raw input), _block, _delta, _flags, _max_loops, _aa_scale, _aa_max_no_dec, _gh_factor,
_strategies (JSON {block_size: [preprocessing block sizes]}, uint8; "{}" = none), _with_u, _status, _b_out, _tours (the
per-tour lines of BKZ_VERBOSE), _lll_out / _lll_status (the wrapper LLL alone, lll_reduction with the same delta; zero
rows first), and with U: _u, _lll_u (the wrapper LLL's own U) and _consistent (whether the reference's U satisfies
U * B_in == B_out over the integers)."""
import io
import json
import os
import re
import subprocess
import sys
import tempfile
import zipfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref")
SHIM = os.path.join(ROOT, "oracle", "shim")
REF_SRC = os.environ.get("REF", "/root/reference")  # the reference sources, as in oracle/Makefile.ref

NO_LLL, MAX_LOOPS, BOUNDED_LLL, AUTO_ABORT, GH_BND, SD, SLD = 2, 4, 0x10, 0x20, 0x80, 0x100, 0x200


def consistent(u, b_in, b_out):
    """U * B_in == B_out over the Python integers"""
    return np.array_equal(np.dot(u.astype(object), b_in.astype(object)), b_out.astype(object))


def rank_deficient(seed, d, n, rank, bits):
    """rank rows of seeded bits-bit entries, then d - rank rows that are small integer combinations of three of them,
    in a seeded row order"""
    rng = np.random.default_rng(seed)
    b = np.zeros((d, n), np.int64)
    b[:rank] = rng.integers(-(1 << bits), 1 << bits, size=(rank, n))
    for i in range(rank, d):
        src = rng.choice(rank, 3, replace=False)
        b[i] = sum(int(rng.integers(-3, 4)) * b[s] for s in src)
    return b[rng.permutation(d)]


def inputs(tmp):
    """the raw input bases, by name"""
    def gen(args):
        p = os.path.join(tmp, "gen.txt")
        open(p, "w").write(O.latticegen(args))
        return np.array(O.read_matrix(p), dtype=np.int64)

    q60 = np.load(os.path.join(HERE, "bkz_q60.npz"))["b_in"]  # latticegen q 60 30 12 b after the reference's wrapper LLL
    rd50 = rank_deficient(3, 50, 50, 46, 16)
    return {
        "q60raw": gen(["q", 60, 30, 12, "b"]),
        "u40": gen(["u", 40, 30]),
        "r80": gen(["r", 80, 40]),
        "q30": gen(["q", 30, 15, 10, "b"]),
        "q60": q60,
        "ns40x60": np.random.default_rng(9).integers(-(1 << 12), 1 << 12, size=(40, 60), dtype=np.int64),
        "rd50": rd50,
        "lz63": np.concatenate([np.zeros((3, 60), np.int64), q60]),
    }


# tag: (input, block, delta, flags, max_loops, (auto_abort_scale, auto_abort_max_no_dec), gh_factor, strategies, with_u)
D = (1.0, 5)
CASES = {
    # the preliminary wrapper LLL of bkz.cpp:869-876 on unreduced inputs, at both deltas
    "plll_q60_d99": ("q60raw", 20, 0.99, MAX_LOOPS, 1, D, 1.1, None, False),
    "plll_q60_d75": ("q60raw", 20, 0.75, MAX_LOOPS, 1, D, 1.1, None, False),
    "plll_u40_d99": ("u40", 10, 0.99, MAX_LOOPS, 1, D, 1.1, None, False),
    "plll_u40_d75": ("u40", 10, 0.75, MAX_LOOPS, 1, D, 1.1, None, False),
    "plll_r80_d99": ("r80", 10, 0.99, MAX_LOOPS, 1, D, 1.1, None, False),
    "plll_r80_d75": ("r80", 10, 0.75, MAX_LOOPS, 1, D, 1.1, None, False),
    "plll_q60_d99_u": ("q60raw", 20, 0.99, MAX_LOOPS, 1, D, 1.1, None, True),
    "plll_r80_d75_u": ("r80", 10, 0.75, MAX_LOOPS, 1, D, 1.1, None, True),
    # runs to convergence (no termination flag); SD-BKZ without one turns auto-abort on (bkz.cpp:548-554)
    "conv_b10": ("q60", 10, 0.99, NO_LLL, 0, D, 1.1, None, False),
    "conv_b20": ("q60", 20, 0.99, NO_LLL, 0, D, 1.1, None, False),
    "conv_sd20": ("q60", 20, 0.99, NO_LLL | SD, 0, D, 1.1, None, False),
    # BKZ_AUTO_ABORT at the default and tighter settings
    "aa_1_5": ("q60", 20, 0.99, NO_LLL | AUTO_ABORT, 0, (1.0, 5), 1.1, None, False),
    "aa_1_1": ("q60", 20, 0.99, NO_LLL | AUTO_ABORT, 0, (1.0, 1), 1.1, None, False),
    "aa_102_2": ("q60", 20, 0.99, NO_LLL | AUTO_ABORT, 0, (1.02, 2), 1.1, None, False),
    "aa_sd_1_2": ("q60", 20, 0.99, NO_LLL | AUTO_ABORT | SD, 0, (1.0, 2), 1.1, None, False),
    # BKZ_GH_BND: applies above block size 30 only; 0.75 is small enough that some blocks find nothing
    "gh30_f075": ("q60", 30, 0.99, NO_LLL | MAX_LOOPS | GH_BND, 1, D, 0.75, None, False),
    "gh32_f110": ("q60", 32, 0.99, NO_LLL | MAX_LOOPS | GH_BND, 1, D, 1.1, None, False),
    "gh36_f075": ("q60", 36, 0.99, NO_LLL | MAX_LOOPS | GH_BND, 1, D, 0.75, None, False),
    "gh40_f110": ("q60", 40, 0.99, NO_LLL | MAX_LOOPS | GH_BND, 1, D, 1.1, None, False),
    # preprocessing without pruning (the preprocessing tours run with BKZ_GH_BND, which applies to their blocks above 30)
    "pre40_20": ("q60", 40, 0.99, NO_LLL | MAX_LOOPS, 1, D, 1.1, {40: [20]}, False),
    "pre30_10_20": ("q60", 30, 0.99, NO_LLL | MAX_LOOPS, 1, D, 1.1, {30: [10, 20], 20: [10]}, False),
    "pre46_34": ("q60", 46, 0.99, NO_LLL | MAX_LOOPS | GH_BND, 1, D, 1.1, {46: [34]}, False),
    "pre40_20_u": ("q60", 40, 0.99, NO_LLL | MAX_LOOPS, 1, D, 1.1, {40: [20]}, True),
    # BKZ_BOUNDED_LLL in BKZ 2.0: svp_preprocessing's LLL starts at kappa
    "bounded20": ("q60", 20, 0.99, NO_LLL | MAX_LOOPS | BOUNDED_LLL, 2, D, 1.1, None, False),
    # block-size edges on a dim-30 basis (to convergence; a block at least the rank is one HKZ pass), non-square
    "edge_b2": ("q30", 2, 0.99, 0, 0, D, 1.1, None, False),
    "edge_b3": ("q30", 3, 0.99, 0, 0, D, 1.1, None, False),
    "edge_b29": ("q30", 29, 0.99, 0, 0, D, 1.1, None, False),
    "edge_b30": ("q30", 30, 0.99, 0, 0, D, 1.1, None, False),
    "edge_b35": ("q30", 35, 0.99, 0, 0, D, 1.1, None, False),
    "ns40x60_b20": ("ns40x60", 20, 0.99, MAX_LOOPS, 2, D, 1.1, None, False),
    # rank-deficient bases: four dependent rows (the wrapper LLL leaves four zero rows), leading zero rows under NO_LLL
    "rd50_plll": ("rd50", 20, 0.99, MAX_LOOPS, 1, D, 1.1, None, False),
    "rd50_plll_u": ("rd50", 20, 0.99, MAX_LOOPS, 1, D, 1.1, None, True),
    "rd50_nolll": ("rd50lll", 20, 0.99, NO_LLL | MAX_LOOPS, 1, D, 1.1, None, False),
    "rd50_sd": ("rd50lll", 10, 0.99, NO_LLL | MAX_LOOPS | SD, 2, D, 1.1, None, False),
    "rd50_sld": ("rd50lll", 10, 0.99, NO_LLL | SLD, 0, D, 1.1, None, False),
    "rd50_b50": ("rd50lll", 50, 0.99, NO_LLL, 0, D, 1.1, None, False),
    "lz63": ("lz63", 20, 0.99, NO_LLL | MAX_LOOPS, 1, D, 1.1, None, False),
    "lz63_u": ("lz63", 20, 0.99, NO_LLL | MAX_LOOPS, 1, D, 1.1, None, True),
}


def strategies_json(strat, block_size):
    """load_strategies_json input: an entry for every block size up to the largest one the call can index (BKZParam
    indexes strategies[block_size], bkz.cpp:89,117), preprocessing block sizes only, no pruning_parameters (so the
    loader fills in PruningParams(), bkz_param.cpp:152-156)"""
    top = max([block_size] + list(strat))
    return json.dumps([{"block_size": k, "preprocessing_block_sizes": [int(x) for x in strat.get(k, [])]}
                       for k in range(top + 1)])


def save_npz(path, arrays):
    """np.savez_compressed with fixed zip timestamps and member order"""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as zf:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            zi = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            zi.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(zi, buf.getvalue())


def main(out_path=None):
    tmp = tempfile.mkdtemp(prefix="bkz_golden_")
    probe = os.path.join(tmp, "bkz_probe")
    inc = ["-I" + os.path.join(SHIM, "include"), "-I" + os.path.join(SHIM, "cfg", "fplll"),
           "-I" + os.path.join(SHIM, "cfg", "fplll", "enum"), "-I" + os.path.join(SHIM, "cfg"), "-I" + REF_SRC,
           "-I" + os.path.join(REF_SRC, "fplll")]
    subprocess.check_call(["g++", "-O2", "-std=c++11", "-pthread"] + inc +
                          [os.path.join(HERE, "bkz_probe.cpp"), "-o", probe, "-L" + REF, "-Wl,-rpath," + REF,
                           "-lfplll", "-l:libmpfr.so.6", "-l:libgmp.so.10"])

    def mat(path):
        return np.array(O.read_matrix(path), dtype=np.int64)

    def run(tag, b_in, bs, delta, fl, ml, aa, ghf, strat, with_u):
        inp, out = os.path.join(tmp, tag + ".in"), os.path.join(tmp, tag)
        O.write_matrix(inp, b_in)
        sp = "-"
        if strat is not None:
            sp = os.path.join(tmp, tag + ".json")
            open(sp, "w").write(strategies_json(strat, bs))
        args = [probe, inp, out, bs, repr(delta), fl, ml, repr(aa[0]), aa[1], repr(ghf), sp, int(with_u)]
        p = subprocess.run([str(a) for a in args], capture_output=True, text=True, timeout=3600)
        if p.returncode != 0:
            raise RuntimeError(tag + ": " + p.stderr[-2000:])
        tok = dict(t.split("=") for t in p.stdout.split())
        rec = {"status": int(tok["status"]), "lll_status": int(tok["lll_status"]), "b_out": mat(out + ".b"),
               "lll_out": mat(out + ".lll"),
               "tours": len(re.findall(r"^End of (?:BKZ|SD-BKZ|SLD) loop", p.stderr, re.M))}
        if with_u:
            rec["u"], rec["lll_u"] = mat(out + ".u"), mat(out + ".lllu")
        return rec

    raw = inputs(tmp)
    # the NO_LLL rank-deficient input: the reference's own wrapper LLL of rd50 (lll_reduction: zero rows first)
    raw["rd50lll"] = run("rd50lll", raw["rd50"], 2, 0.99, MAX_LOOPS, 0, D, 1.1, None, False)["lll_out"]

    def one(item):
        tag, (src, bs, delta, fl, ml, aa, ghf, strat, with_u) = item
        return tag, run(tag, raw[src], bs, delta, fl, ml, aa, ghf, strat, with_u)

    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        results = dict(ex.map(one, sorted(CASES.items())))
    pack = {}
    for tag in sorted(CASES):
        src, bs, delta, fl, ml, aa, ghf, strat, with_u = CASES[tag]
        r = results[tag]
        pack.update({tag + "_b_in": raw[src], tag + "_block": np.int32(bs), tag + "_delta": np.float64(delta),
                     tag + "_flags": np.int32(fl), tag + "_max_loops": np.int32(ml),
                     tag + "_aa_scale": np.float64(aa[0]), tag + "_aa_max_no_dec": np.int32(aa[1]),
                     tag + "_gh_factor": np.float64(ghf),
                     tag + "_strategies": np.frombuffer(json.dumps({str(k): v for k, v in sorted((strat or {}).items())})
                                                        .encode(), np.uint8),
                     tag + "_with_u": np.bool_(with_u), tag + "_status": np.int32(r["status"]),
                     tag + "_b_out": r["b_out"], tag + "_tours": np.int32(r["tours"]),
                     tag + "_lll_out": r["lll_out"], tag + "_lll_status": np.int32(r["lll_status"])})
        if with_u:
            pack[tag + "_u"], pack[tag + "_lll_u"] = r["u"], r["lll_u"]
            pack[tag + "_consistent"] = np.bool_(consistent(r["u"], raw[src], r["b_out"]))
        print("%-14s status %d tours %d%s" % (tag, r["status"], r["tours"],
                                              " U consistent %s" % bool(pack[tag + "_consistent"]) if with_u else ""),
              flush=True)
    pack["tags"] = np.frombuffer(json.dumps(sorted(CASES)).encode(), np.uint8)
    save_npz(out_path or os.path.join(HERE, "bkz_driver_ref.npz"), pack)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
