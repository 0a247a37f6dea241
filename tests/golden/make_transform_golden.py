"""Regenerates tests/golden/transform_ref.npz: the transform U the UNMODIFIED reference computes next to b (MatGSO with a
non-empty u; bkz_reduction with a non-empty U), from the reference build in oracle/_ref (oracle/Makefile.ref).  Run in the
build container only, after that build:
    python tests/golden/make_transform_golden.py [OUT.npz]
It compiles transform_probe.cpp (next to this file) into a temporary directory and runs it; ~1 min of CPU.

Cases (prefix -> what):
  ops<k>    seeded op scripts on the u 40 input of config #1 (u40_lll_long.npz), GSO_ROW_EXPO | GSO_OP_FORCE_LONG: groups
            of row_addmul_we (with 2^e shifts, some of them wrapping), row_swap, move_row in both directions and negate_row_of_b, each group closed by
            update_gso; U after every group (ops<k>_u[g]) and b after the last one
  lll_u40   LLL<long, double> (GSO_ROW_EXPO) on u40_lll_long.npz:b_in
  lll_r200  LLL<long, double> on a seeded dim-200 knapsack basis (40-bit weights)
  lll_rankdef  LLL<long, double> on a seeded 40 x 41 basis of rank 30 (ten rows are integer combinations of others, so LLL
            ends with ten zero rows and U is not determined by B)
  bkz20 / sd20 / sld20  bkz_reduction(b, u, BKZParam(20), FT_DOUBLE) without pruning on bkz_q60.npz:b_in, with the flags
            of the existing goldens (bkz_q60.npz bkz20_none, bkz_sd_sld.npz sd20_none / sld20_none)
Every case records <tag>_consistent: whether the reference's own U satisfies U * B_in == B_out over the integers (the
reference's negate_row_of_b leaves u alone, so after a negation it does not)."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref")
SHIM = os.path.join(ROOT, "oracle", "shim")
REF_SRC = os.environ.get("REF", "/root/reference")  # the reference sources, as in oracle/Makefile.ref


def op_script(rng, d, n_groups, per_group):
    """Groups of row operations for a transform test: ["addmul", i, j, x, e], ["swap", i, j], ["move", old, new],
    ["negate", i].  Negations only in the second half, so that U can be compared with the reference's for half the
    script; a few addmuls carry an exponent that makes row_addmul_we shift (and wrap) the products."""
    groups = []
    for g in range(n_groups):
        ops = []
        for _ in range(per_group):
            k = int(rng.integers(0, 10 if g >= n_groups // 2 else 9))
            if k < 4:
                i, j = (int(t) for t in rng.choice(d, 2, replace=False))
                ops.append(["addmul", i, j, float(rng.integers(-9, 10)), 0])
            elif k < 6:
                i, j = (int(t) for t in rng.choice(d, 2, replace=False))
                ops.append(["addmul", i, j, float(rng.integers(-3, 4)), int(rng.integers(1, 4))])
            elif k == 6:
                i, j = (int(t) for t in rng.choice(d, 2, replace=False))
                ops.append(["addmul", i, j, float(rng.choice([-7, 3, 5])), int(rng.choice([61, 62]))])
            elif k == 7:
                i, j = sorted(int(t) for t in rng.choice(d, 2, replace=False))
                ops.append(["swap", i, j])
            elif k == 8:
                a, b = (int(t) for t in rng.choice(d, 2, replace=False))
                ops.append(["move", a, b])
            else:
                ops.append(["negate", int(rng.integers(0, d))])
        groups.append(ops)
    return groups


def op_lines(op):
    k, a = op[0], op[1:]
    if k == "addmul":
        return ["row_op_begin %d %d" % (a[0], a[0] + 1), "row_addmul_we %d %d %r %d" % tuple(a),
                "row_op_end %d %d" % (a[0], a[0] + 1)]
    if k == "swap":
        return ["row_op_begin %d %d" % (a[0], a[1] + 1), "row_swap %d %d" % tuple(a), "row_op_end %d %d" % (a[0], a[1] + 1)]
    if k == "move":
        return ["move_row %d %d" % tuple(a)]
    return ["row_op_begin %d %d" % (a[0], a[0] + 1), "negate %d" % a[0], "row_op_end %d %d" % (a[0], a[0] + 1)]


def consistent(u, b_in, b_out):
    """U * B_in == B_out over the Python integers"""
    U = [[int(x) for x in row] for row in u]
    Bi = [[int(x) for x in row] for row in b_in]
    for i, row in enumerate(U):
        for c in range(len(Bi[0])):
            if sum(row[k] * Bi[k][c] for k in range(len(Bi))) != int(b_out[i][c]):
                return False
    return True


def knapsack(seed, d, bits):
    rng = np.random.default_rng(seed)
    b = np.zeros((d, d + 1), np.int64)
    b[:, 0] = rng.integers(1, 1 << bits, size=d)
    b[:, 1:] = np.eye(d, dtype=np.int64)
    return b


def rank_deficient(seed, d, n, rank):
    rng = np.random.default_rng(seed)
    b = np.zeros((d, n), np.int64)
    b[:rank] = rng.integers(-(1 << 20), 1 << 20, size=(rank, n))
    for i in range(rank, d):
        src = rng.choice(rank, 3, replace=False)
        b[i] = sum(int(rng.integers(-3, 4)) * b[s] for s in src)
    return b[rng.permutation(d)]


def main(out_path=None):
    tmp = tempfile.mkdtemp(prefix="transform_golden_")
    probe = os.path.join(tmp, "transform_probe")
    inc = ["-I" + os.path.join(SHIM, "include"), "-I" + os.path.join(SHIM, "cfg", "fplll"),
           "-I" + os.path.join(SHIM, "cfg", "fplll", "enum"), "-I" + os.path.join(SHIM, "cfg"), "-I" + REF_SRC,
           "-I" + os.path.join(REF_SRC, "fplll")]
    subprocess.check_call(["g++", "-O2", "-std=c++11", "-pthread"] + inc +
                          [os.path.join(HERE, "transform_probe.cpp"), "-o", probe, "-L" + REF, "-Wl,-rpath," + REF,
                           "-lfplll", "-l:libmpfr.so.6", "-l:libgmp.so.10"])

    def run(script):
        p = subprocess.run([probe], input=script, capture_output=True, text=True, timeout=3600)
        if p.returncode != 0:
            raise RuntimeError(p.stderr[-2000:])
        return p.stdout

    def mat(path):
        return np.array(O.read_matrix(path), dtype=np.int64)

    pack = {}
    u40 = np.load(os.path.join(HERE, "u40_lll_long.npz"))["b_in"]
    inp = os.path.join(tmp, "in.txt")
    # op scripts
    for k, seed in enumerate((11, 12)):
        groups = op_script(np.random.default_rng(seed), u40.shape[0], 12, 8)
        O.write_matrix(inp, u40)
        # GSO_ROW_EXPO | GSO_OP_FORCE_LONG: the shifted products go through row_addmul_si_2exp, the int64 arithmetic the
        # device implements (include/b200gso.h: GSO_OP_FORCE_LONG is implied there)
        lines = ["load " + inp, "gso 6", "update_gso"]
        for g, ops in enumerate(groups):
            for op in ops:
                lines += op_lines(op)
            lines += ["update_gso", "save_u %s/u_%d.txt" % (tmp, g)]
        lines.append("save_b %s/b.txt" % tmp)
        run("\n".join(lines) + "\n")
        us = np.stack([mat("%s/u_%d.txt" % (tmp, g)) for g in range(len(groups))])
        b_out = mat(tmp + "/b.txt")
        pack["ops%d_script" % k] = np.frombuffer(json.dumps(groups).encode(), np.uint8)
        pack["ops%d_b_in" % k] = u40
        pack["ops%d_u" % k] = us
        pack["ops%d_b_out" % k] = b_out
        pack["ops%d_consistent" % k] = np.bool_(consistent(us[-1], u40, b_out))
        first_neg = min((g for g, ops in enumerate(groups) if any(o[0] == "negate" for o in ops)), default=len(groups))
        print("ops%d: first negation in group %d, reference U consistent at the end: %s"
              % (k, first_neg, bool(pack["ops%d_consistent" % k])), flush=True)
    # LLL
    for tag, b_in in (("lll_u40", u40), ("lll_r200", knapsack(7, 200, 40)), ("lll_rankdef", rank_deficient(5, 40, 41, 30))):
        O.write_matrix(inp, b_in)
        o = run("load %s\ngso 2\nlll 0.99 0.51\nsave_b %s/b.txt\nsave_u %s/u.txt\n" % (inp, tmp, tmp))
        tok = dict(t.split("=") for t in o.split("lll ")[1].split())
        b_out, u = mat(tmp + "/b.txt"), mat(tmp + "/u.txt")
        pack.update({tag + "_b_in": b_in, tag + "_b_out": b_out, tag + "_u": u, tag + "_status": np.int32(tok["status"]),
                     tag + "_swaps": np.int32(tok["swaps"]), tag + "_zeros": np.int32(tok["zeros"]),
                     tag + "_consistent": np.bool_(consistent(u, b_in, b_out))})
        print(tag, o.strip(), "consistent", bool(pack[tag + "_consistent"]), flush=True)
    # BKZ without pruning
    q60 = np.load(os.path.join(HERE, "bkz_q60.npz"))["b_in"]
    NO_LLL, MAX_LOOPS, SD, SLD = 2, 4, 0x100, 0x200
    for tag, fl, ml in (("bkz20", NO_LLL, 0), ("sd20", SD | NO_LLL | MAX_LOOPS, 2), ("sld20", SLD | NO_LLL, 0)):
        O.write_matrix(inp, q60)
        o = run("load %s\nbkz 20 %d %d\nsave_b %s/b.txt\nsave_u %s/u.txt\n" % (inp, fl, ml, tmp, tmp))
        b_out, u = mat(tmp + "/b.txt"), mat(tmp + "/u.txt")
        pack.update({tag + "_b_out": b_out, tag + "_u": u, tag + "_flags": np.int32(fl), tag + "_max_loops": np.int32(ml),
                     tag + "_status": np.int32(int(o.split("bkz status=")[1].split()[0])),
                     tag + "_consistent": np.bool_(consistent(u, q60, b_out))})
        print(tag, o.strip(), "consistent", bool(pack[tag + "_consistent"]), flush=True)
    pack["q60_b_in"] = q60
    np.savez_compressed(out_path or os.path.join(HERE, "transform_ref.npz"), **pack)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
