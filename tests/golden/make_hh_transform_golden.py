"""Regenerates tests/golden/hh_transform_ref.npz: the transform U and U^-T the UNMODIFIED reference computes next to b in
MatHouseholder<Z_NR<long>, FP_NR<double>> (u and u_inv_t non-empty) and in HLLLReduction<Z_NR<long>, FP_NR<double>>
with HOUSEHOLDER_ROW_EXPO | HOUSEHOLDER_OP_FORCE_LONG, from the reference build in oracle/_ref (oracle/Makefile.ref).
Run in the build container only, after that build:
    python tests/golden/make_hh_transform_golden.py [OUT.npz]
It compiles hh_transform_probe.cpp (next to this file) into a temporary directory and runs it; ~1 min of CPU.

Cases: `cases` (JSON) lists every whole-HLLL case as tag -> the fixture and key its input comes from ("self" = stored
here as <tag>_in); each has <tag>_out, <tag>_status, <tag>_u and <tag>_uinvt (U^-T as the reference's object holds
it: hlll_reduction(b, u, u_inv) returns its transpose, U^-1).
  u40 r60 q40 u100 q80   hlll_long.npz inputs
  q400sub                hlll_q400.npz (120 x 400 rows of BASELINE config #3)
  hlll600                size_classes_ref.npz (30 x 600)
  mix170                 seeded 170 x 180 basis, small random combinations of random rows (170 is not a multiple of
                         32: a row of U spans six lane rounds, the last one partial)
and one call script, script_*: the hh_* calls of tests/test_hh_gpu.py::_hlll_like_ops on a seeded 24 x 30 basis
(script_in, script_ops as JSON), with b, U and U^-T at every check point (script_b, script_u, script_uinvt)."""
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

CASES = {"u40": "hlll_long.npz:u40_in", "r60": "hlll_long.npz:r60_in", "q40": "hlll_long.npz:q40_in",
         "u100": "hlll_long.npz:u100_in", "q80": "hlll_long.npz:q80_in", "q400sub": "hlll_q400.npz:q400sub_in",
         "hlll600": "size_classes_ref.npz:hlll600_in", "mix170": "self"}
SCRIPT_SEED, SCRIPT_D, SCRIPT_N, SCRIPT_BITS = 21, 24, 30, 30


def mix170():
    rng = np.random.default_rng(170)
    u = rng.integers(-8, 9, size=(170, 170), dtype=np.int64)
    return u @ rng.integers(-(1 << 10), 1 << 10, size=(170, 180), dtype=np.int64)


def hlll_like_ops(d):
    """tests/test_hh_gpu.py::_hlll_like_ops: HLLLReduction::hlll's call order (hlll.cpp:49-171) with a swap every
    third step"""
    ops = [("refresh_R_bf", 0), ("update_R_last", 0), ("refresh_R_bf", 1)]
    k, kmax = 1, 1
    for step in range(3 * d):
        ops += [("update_R", k, 0), ("size_reduce", k, k, 0), ("refresh_R_bf", k), ("update_R", k, 0), ("check",)]
        if step % 3 != 2 or k == 1:
            ops += [("update_R_last", k)]
            k += 1
            if k >= d:
                break
            ops += [("refresh_R_bf", k)] if k > kmax else [("refresh_R", k)]
            kmax = max(kmax, k)
        else:
            ops += [("swap", k - 1, k)]
            k -= 1
            ops += [("recover_R", k), ("check",), ("set_updated_R_false",)]
    ops.append(("check",))
    return ops


def script_input():
    rng = np.random.default_rng(SCRIPT_SEED)
    return rng.integers(-(1 << SCRIPT_BITS), 1 << SCRIPT_BITS, size=(SCRIPT_D, SCRIPT_N), dtype=np.int64)


def load_input(src):
    f, k = src.split(":")
    return np.load(os.path.join(HERE, f))[k].astype(np.int64)


def main(out_path=None):
    tmp = tempfile.mkdtemp(prefix="hh_transform_golden_")
    probe = os.path.join(tmp, "hh_transform_probe")
    inc = ["-I" + os.path.join(SHIM, "include"), "-I" + os.path.join(SHIM, "cfg", "fplll"),
           "-I" + os.path.join(SHIM, "cfg", "fplll", "enum"), "-I" + os.path.join(SHIM, "cfg"), "-I" + REF_SRC,
           "-I" + os.path.join(REF_SRC, "fplll")]
    subprocess.check_call(["g++", "-O2", "-std=c++11", "-pthread"] + inc +
                          [os.path.join(HERE, "hh_transform_probe.cpp"), "-o", probe, "-L" + REF, "-Wl,-rpath," + REF,
                           "-lfplll", "-l:libmpfr.so.6", "-l:libgmp.so.10"])

    def run(script):
        p = subprocess.run([probe], input=script, capture_output=True, text=True, timeout=3600)
        if p.returncode != 0:
            raise RuntimeError(p.stderr[-2000:])
        return p.stdout

    def mat(path):
        return np.array(O.read_matrix(path), dtype=np.int64)

    pack = {"cases": np.frombuffer(json.dumps(CASES).encode(), np.uint8)}
    inp = os.path.join(tmp, "in.txt")
    for tag, src in CASES.items():
        b_in = mix170() if src == "self" else load_input(src)
        if src == "self":
            pack[tag + "_in"] = b_in
        O.write_matrix(inp, b_in)
        o = run("load %s\nhlll 0.99 0.51 0.001 0.1\nsave_b %s/b.txt\nsave_u %s/u.txt\nsave_uinvt %s/ut.txt\n"
                % (inp, tmp, tmp, tmp))
        pack[tag + "_status"] = np.int32(int(o.split("hlll status=")[1].split()[0]))
        pack[tag + "_out"], pack[tag + "_u"], pack[tag + "_uinvt"] = (mat("%s/%s.txt" % (tmp, f)) for f in ("b", "u", "ut"))
        print(tag, b_in.shape, "status", int(pack[tag + "_status"]), "max |U|", int(np.abs(pack[tag + "_u"]).max()),
              flush=True)
    # the call script, U and U^-T at every check point
    b = script_input()
    ops = hlll_like_ops(SCRIPT_D)
    O.write_matrix(inp, b)
    lines, checks = ["load " + inp, "hh %d" % (O.HOUSEHOLDER_ROW_EXPO | O.HOUSEHOLDER_OP_FORCE_LONG)], 0
    for op in ops:
        if op[0] == "check":
            lines += ["save_%s %s/%s_%d.txt" % (w, tmp, w, checks) for w in ("b", "u", "uinvt")]
            checks += 1
        else:
            lines.append("hh_%s %s" % (op[0], " ".join(str(a) for a in op[1:])))
    run("\n".join(lines) + "\n")
    pack["script_in"] = b
    pack["script_ops"] = np.frombuffer(json.dumps(ops).encode(), np.uint8)
    for w in ("b", "u", "uinvt"):
        pack["script_" + w] = np.stack([mat("%s/%s_%d.txt" % (tmp, w, t)) for t in range(checks)])
    print("script: %d checks" % checks, flush=True)
    np.savez_compressed(out_path or os.path.join(HERE, "hh_transform_ref.npz"), **pack)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
