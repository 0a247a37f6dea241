"""Regenerates tests/golden/*.npz from the UNMODIFIED reference (oracle/_ref, built from /root/reference by
oracle/Makefile.ref).  Run in the build container only:  python tests/golden/make_golden.py
Inputs come from the reference's own latticegen (default seed), never from a re-implementation (SURVEY §8c)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import oracle as O  # noqa: E402
import helpers as H  # noqa: E402

TMP = "/tmp/lat"
os.makedirs(TMP, exist_ok=True)


def save_state(path, rec, extra=None):
    keys = ["d", "n", "n_known_rows", "n_known_cols", "n_source_rows", "flags", "row_expo", "gso_valid_cols",
            "init_row_size", "bf", "gf", "mu", "r", "b"]
    out = {k: rec[k] for k in keys if k in rec}
    out.update(extra or {})
    np.savez_compressed(path, **out)


def gen(args, name):
    p = os.path.join(TMP, name)
    if not os.path.exists(p):
        open(p, "w").write(O.latticegen(args))
    return p


def bkz_fixtures():
    # --- BKZ fixtures: q-ary dim-60 (latticegen q 60 30 12 b), reference wrapper-LLL, then reference BKZ ----------
    q60 = gen(["q", 60, 30, 12, "b"], "q60.txt")
    q60l = os.path.join(TMP, "q60_lll.txt")
    O.run_ref("load %s\nlll 0.99 0.51 wrapper default 0\nsave %s\n" % (q60, q60l))
    b_in = np.array(O.read_matrix(q60l), dtype=np.int64)
    pack = {"b_in": b_in}
    # (block, flags, max_loops, strategies): BKZ_NO_LLL = 2, BKZ_MAX_LOOPS = 4
    for tag, bs, fl, ml, strat in [("bkz20_none", 20, 2, 0, "none"), ("bkz30_default", 30, 2 | 4, 2, "default"),
                                   ("bkz40_default", 40, 2 | 4, 2, "default")]:
        outp = os.path.join(TMP, "q60_%s.txt" % tag)
        o = O.run_ref("load %s\nbkz %d %d %d %s enumlib 1\nsave %s\n" % (q60l, bs, fl, ml, strat, outp), timeout=600)
        st = int(o.split("bkz status=")[1].split()[0])
        pack[tag + "_status"] = np.int32(st)
        pack[tag + "_b"] = np.array(O.read_matrix(outp), dtype=np.int64)
    np.savez_compressed(os.path.join(HERE, "bkz_q60.npz"), **pack)


def hlll_fixtures():
    # --- HLLL fixtures: the reference's HLLLReduction<long,double>::hlll (ROW_EXPO | OP_FORCE_LONG, defaults
    # delta 0.99, eta 0.51, theta 0.001, c 0.1) on latticegen inputs that fit int64 -------------------------------
    pack = {}
    for tag, args in [("u40", ["u", 40, 16]), ("r60", ["r", 60, 55]), ("q40", ["q", 40, 20, 12, "b"]),
                      ("u100", ["u", 100, 20]), ("q80", ["q", 80, 40, 16, "b"])]:
        inp = gen(args, "hlll_%s.txt" % tag)
        outp = os.path.join(TMP, "hlll_%s_out.txt" % tag)
        o = O.run_ref("load %s\ntolong\nhlll_long 0.99 0.51 0.001 0.1\nsave_long %s\n" % (inp, outp), timeout=600)
        pack[tag + "_in"] = np.array(O.read_matrix(inp), dtype=np.int64)
        pack[tag + "_out"] = np.array(O.read_matrix(outp), dtype=np.int64)
        pack[tag + "_status"] = np.int32(int(o.split("hlll_long status=")[1].split()[0]))
    np.savez_compressed(os.path.join(HERE, "hlll_long.npz"), **pack)


def svp_kat_fixture():
    # --- the reference's SVP known-answer pair (tests/test_svp.cpp:373-374): input basis and a shortest vector -------
    import re
    src = "/root/reference/tests/lattices/"
    rows = re.findall(r"\[([^\[\]]*)\]", open(src + "example_svp_in").read())
    b = np.array([[int(x) for x in r.split()] for r in rows if r.strip()], dtype=np.int64)
    sv = np.array([int(x) for x in re.findall(r"-?\d+", open(src + "example_svp_out").read())], dtype=np.int64)
    np.savez_compressed(os.path.join(HERE, "example_svp.npz"), b_in=b, sv=sv)


def main():
    if '--only-svp' in sys.argv:
        return svp_kat_fixture()
    if '--only-bkz' in sys.argv:
        return bkz_fixtures()
    if '--only-hlll' in sys.argv:
        return hlll_fixtures()
    # --- config #1 input: latticegen u 40 40 (md5 a6fe01e1..., BASELINE.md) -------------------------------
    u40 = np.array(O.read_matrix(gen(["u", 40, 40], "u40.txt")), dtype=np.int64)
    s = O.RefSession(u40)
    s.cmd("update_gso")
    s.dump_state()
    _, recs = s.run()
    save_state(os.path.join(HERE, "u40_update_gso.npz"), recs[0])

    # op-sequence trace on u40 (state machine: row ops, move_row, partial updates), dumped after every op group
    rng = np.random.default_rng(20260923)
    ops = H.random_op_script(rng, 40, 60)
    s = O.RefSession(u40)
    marks = []
    for k, op in enumerate(ops):
        for line in H.ops_to_ref_script([op]):
            s.lines.append(line)
        if op[0] in ("move_row", "update_gso") or (op[0] in ("row_op_end", "update_rows_to") and k % 3 == 0):
            s.dump_state()
            marks.append(k)
    _, recs = s.run()
    assert len(recs) == len(marks)
    import json
    pack = {"ops_json": np.frombuffer(json.dumps(ops).encode(), dtype=np.uint8), "marks": np.array(marks),
            "b0": u40}
    for t, r in enumerate(recs):
        for key in ["n_known_rows", "n_known_cols", "n_source_rows"]:
            pack["s%d_%s" % (t, key)] = np.int32(r[key])
        for key in ["row_expo", "gso_valid_cols", "init_row_size", "bf", "gf", "mu", "r", "b"]:
            pack["s%d_%s" % (t, key)] = r[key]
    np.savez_compressed(os.path.join(HERE, "u40_ops_trace.npz"), **pack)

    # reference LLL on u40 through the <long,double> code path (MatGSO<long,double>+LLLReduction, GSO_ROW_EXPO)
    mat = os.path.join(TMP, "u40.txt")
    out = O.run_ref("load %s\ntolong\nlll_long 0.99 0.51\ngso l 2\nsave %s/u40_lll_long.txt\n" % (mat, TMP))
    st = dict(tok.split("=") for tok in out.split("lll_long")[1].split() if "=" in tok)
    red = np.array(O.read_matrix(TMP + "/u40_lll_long.txt"), dtype=np.int64)
    np.savez_compressed(os.path.join(HERE, "u40_lll_long.npz"), b_in=u40, b_out=red, status=np.int32(st["status"]),
                        n_swaps=np.int32(st["swaps"]))

    # --- config #2/#5 input after the host wrapper LLL (bkz.cpp:873-875): int64 regime dim-200 -------------
    r200 = gen(["r", 200, 2000], "r200.txt")
    red_path = os.path.join(TMP, "r200_lll.txt")
    if not os.path.exists(red_path):
        O.run_ref("load %s\nlll 0.99 0.51 wrapper default 0\nsave %s\n" % (r200, red_path), timeout=900)
    b200 = np.array(O.read_matrix(red_path), dtype=np.int64)
    s = O.RefSession(b200)
    s.cmd("update_gso")
    s.dump_state()
    _, recs = s.run()
    rec = recs[0]
    # keep the fixture small: b + the derived state in compact form (mu/r lower triangles as float64)
    tl = np.tril_indices(200)
    np.savez_compressed(os.path.join(HERE, "r200_lll_update_gso.npz"), b=b200, row_expo=rec["row_expo"],
                        gso_valid_cols=rec["gso_valid_cols"], init_row_size=rec["init_row_size"],
                        n_known_rows=np.int32(rec["n_known_rows"]), n_known_cols=np.int32(rec["n_known_cols"]),
                        n_source_rows=np.int32(rec["n_source_rows"]),
                        mu_tril=rec["mu"][tl], r_tril=rec["r"][tl], gf_tril=rec["gf"][tl])
    # --- enumeration fixtures (reference's internal enumerator through the plugin-API capture hook) ----------
    import json
    strat = json.load(open(os.path.join(O.REF_DIR, "strategies", "default.json")))
    s60 = [e for e in strat if e["block_size"] == 60][0]
    pr60 = s60["pruning_parameters"][15]   # [gh_factor = 1.05, coefficients, probability ~ 0.41]
    prfile = os.path.join(TMP, "prune60.txt")
    open(prfile, "w").write(" ".join(repr(float(c)) for c in pr60[1]))
    out = os.path.join(TMP, "enum_fixture.bin")
    if os.path.exists(out):
        os.remove(out)
    # radius as BKZ sets it (bkz.cpp:310-323): gh_factor * GH^2 of the block, expressed as a multiple of r(first,first)
    import math
    Rm = np.zeros((200, 200))
    Rm[tl] = rec["r"][tl]
    rii = np.array([Rm[i, i] * 2.0 ** (2 * int(rec["row_expo"][i])) for i in range(200)])

    def gh_ratio(first, last):
        n = last - first
        gh2 = math.exp((2.0 / n) * math.lgamma(n / 2 + 1)) / math.pi * math.exp(np.sum(np.log(rii[first:last])) / n)
        return gh2 / rii[first]
    f100, f140 = float(1.05 * gh_ratio(100, 160)), float(1.05 * gh_ratio(140, 200))
    script = ("load %s\ntolong\ngso l 2\nupdate_gso\n"
              "enum 0 30 0.99 - %s capture\n"
              "enum 100 160 %r %s %s capture\n"
              "enum 140 200 %r %s %s capture\n") % (red_path, out, f100, prfile, out, f140, prfile, out)
    print(O.run_ref(script, timeout=600))
    recs = O.read_enum_records(out)
    for name, r in zip(["enum_r200_b30_unpruned", "enum_r200_b60_pruned_100", "enum_r200_b60_pruned_140"], recs):
        np.savez_compressed(os.path.join(HERE, name + ".npz"), mut=r["mut"], rdiag=r["rdiag"], pruning=r["pruning"],
                            maxdist=np.float64(r["maxdist"]), normexp=np.int64(r["normexp"]),
                            found=np.int32(r["found"]), best=np.float64(r["best"]), sol=r["sol"], nodes=r["nodes"],
                            gh_factor=np.float64(pr60[0]))
    # Leech lattice known-answer test (tests/test_enum.cpp:55-100): 196560 minimal vectors of squared norm 32
    leech_in = "/root/reference/tests/lattices/example_list_cvp_in_lattice"
    lo = os.path.join(TMP, "leech_lll.txt")
    O.run_ref("load %s\nlll 0.99 0.51 wrapper default 0\nsave %s\n" % (leech_in, lo))
    np.savez_compressed(os.path.join(HERE, "leech_lll.npz"), b=np.array(O.read_matrix(lo), dtype=np.int64))
    bkz_fixtures()
    hlll_fixtures()
    svp_kat_fixture()
    print("golden fixtures written to", HERE)


def config_size_fixtures():
    """BASELINE.json configs #3-#5 at their stated sizes (python tests/golden/make_golden.py --configs; ~25 min of CPU):
      #3 HLLL on latticegen q 400 200 30 b: the reference's HLLLReduction<long,double> on the full 400 x 400 basis
         (status + output) and on the 120-row sub-lattice rows [140, 260) (a case a test can afford on every run);
      #4 BKZ-40 on the dim-180 Goldstein-Mayer basis (latticegen q 180 1 1800 p), wrapper-LLL first (bkz.cpp:869-876),
         no pruning => deterministic => the output basis is the known answer;
      #5 BKZ-60 with strategies/default.json, one tour, on the LLL-reduced r200 basis: status, r(0,0) and slope."""
    import time
    pack = {}
    q400 = gen(["q", 400, 200, 30, "b"], "q400.txt")
    b400 = np.array(O.read_matrix(q400), dtype=np.int64)
    sub = os.path.join(TMP, "q400_rows140_260.txt")
    O.write_matrix(sub, b400[140:260])
    for tag, inp in (("q400sub", sub), ("q400", q400)):
        outp = os.path.join(TMP, "hlll_%s_out.txt" % tag)
        t0 = time.time()
        o = O.run_ref("load %s\ntolong\nhlll_long 0.99 0.51 0.001 0.1\nsave_long %s\n" % (inp, outp), timeout=7200)
        pack[tag + "_hlll_sec"] = np.float64(time.time() - t0)
        pack[tag + "_in"] = np.array(O.read_matrix(inp), dtype=np.int64)
        pack[tag + "_out"] = np.array(O.read_matrix(outp), dtype=np.int64)
        pack[tag + "_status"] = np.int32(int(o.split("hlll_long status=")[1].split()[0]))
        print(tag, "hlll status", pack[tag + "_status"], "sec", pack[tag + "_hlll_sec"], flush=True)
    del pack["q400_in"], pack["q400_out"]  # the full run ends in status 10 after minutes: keep its status and time only
    np.savez_compressed(os.path.join(HERE, "hlll_q400.npz"), **pack)
    pack = {}
    gm = gen(["q", 180, 1, 1800, "p"], "gm180.txt")
    gml = os.path.join(TMP, "gm180_lll.txt")
    O.run_ref("load %s\nlll 0.99 0.51 wrapper default 0\nsave %s\n" % (gm, gml), timeout=3600)
    pack["b_in"] = np.array(O.read_matrix(gml), dtype=np.int64)
    outp = os.path.join(TMP, "gm180_bkz40.txt")
    t0 = time.time()
    o = O.run_ref("load %s\nbkz 40 %d 1 none enumlib 1\nsave %s\n" % (gml, 2 | 4, outp), timeout=7200)
    pack["bkz40_none_sec"] = np.float64(time.time() - t0)
    pack["bkz40_none_status"] = np.int32(int(o.split("bkz status=")[1].split()[0]))
    pack["bkz40_none_b"] = np.array(O.read_matrix(outp), dtype=np.int64)
    print("gm180 bkz40 status", pack["bkz40_none_status"], "sec", pack["bkz40_none_sec"], flush=True)
    np.savez_compressed(os.path.join(HERE, "bkz_gm180.npz"), **pack)
    g = np.load(os.path.join(HERE, "r200_lll_update_gso.npz"))
    mat = os.path.join(TMP, "r200_red.txt")
    O.write_matrix(mat, g["b"])
    outp = os.path.join(TMP, "r200_bkz60.txt")
    o = O.run_ref("load %s\nbkz 60 %d 1 default enumlib 1\nsave %s\n" % (mat, 2 | 4, outp), timeout=7200)
    b = np.array(O.read_matrix(outp), dtype=np.int64)
    np.savez_compressed(os.path.join(HERE, "bkz60_r200_ref.npz"), status=np.int32(int(o.split("bkz status=")[1].split()[0])),
                        b_out=b)
    print(o, flush=True)


def enum_dual_subsol_fixtures():
    """Dual SVP enumeration and sub-solutions (SURVEY §8 f4): block [140,170) of the LLL-reduced r200 basis, unpruned,
    through the capture hook (records what the plugin API hands an external enumerator, then the reference's own
    enumerator runs).  Standalone: python tests/golden/make_golden.py --dual"""
    g = np.load(os.path.join(HERE, "r200_lll_update_gso.npz"))
    os.makedirs(TMP, exist_ok=True)
    mat = os.path.join(TMP, "r200_red.txt")
    O.write_matrix(mat, g["b"])
    out = os.path.join(TMP, "enum_dual_fixture.bin")
    if os.path.exists(out):
        os.remove(out)
    modes = ["capture", "capture_dual", "capture_subsols", "capture_dual_subsols"]
    script = "load %s\ntolong\ngso l 2\nupdate_gso\n" % mat + "".join(
        "enum 140 170 0.99 - %s %s\n" % (out, m) for m in modes)
    print(O.run_ref(script, timeout=600))
    recs = O.read_enum_records(out)
    arrs = dict(mut=recs[0]["mut"], rdiag=recs[0]["rdiag"], pruning=recs[0]["pruning"])
    for m, r in zip(["primal", "dual", "subsols", "dual_subsols"], recs):
        assert np.array_equal(r["mut"], recs[0]["mut"]) and np.array_equal(r["rdiag"], recs[0]["rdiag"])
        arrs[m + "_maxdist"] = np.float64(r["maxdist"])
        arrs[m + "_best"] = np.float64(r["best"])
        arrs[m + "_normexp"] = np.int64(r["normexp"])
        arrs[m + "_sol"] = r["sol"]
        arrs[m + "_nodes"] = r["nodes"]
        if r["subsols"]:
            arrs[m + "_subdist"] = r["subdist"]
            arrs[m + "_subsol"] = r["subsol"]
    np.savez_compressed(os.path.join(HERE, "enum_r200_b30_dual_subsols.npz"), **arrs)


def config2_mpz_reference():
    """BASELINE config #2 as written (LLL<mpz_t,double> on latticegen r 200 2000): the reference's own outcome — status,
    GSO dump and basis of tests/shim_demo without the shim — as hashes in lll_r200_mpz_ref.json (33 s on one core)."""
    import hashlib
    import json
    import subprocess
    root = os.path.dirname(os.path.dirname(HERE))
    inp, out = os.path.join(TMP, "r200.txt"), os.path.join(TMP, "r200_out.bin")
    open(inp, "w").write(O.latticegen(["r", 200, 2000]))
    env = dict(os.environ, LD_LIBRARY_PATH=os.path.join(root, "oracle", "_ref"))
    env.pop("LD_PRELOAD", None)
    p = subprocess.run([os.path.join(root, "tests", "_build", "shim_demo"), inp, "mpz", out], capture_output=True,
                       text=True, env=env, timeout=900)
    tok = dict(t.split("=") for t in p.stdout.split() if "=" in t)
    sha = lambda f: hashlib.sha256(open(f, "rb").read()).hexdigest()
    rec = dict(what="BASELINE config #2: reference LLLReduction<Z_NR<mpz_t>, FP_NR<double>> on latticegen r 200 2000",
               made_by="tests/golden/make_golden.py::config2_mpz_reference",
               input_md5=hashlib.md5(open(inp, "rb").read()).hexdigest(), status=int(tok["status"]),
               gso_ok=int(tok["gso_ok"]), out_bin_sha256=sha(out), out_basis_sha256=sha(out + ".basis"))
    json.dump(rec, open(os.path.join(HERE, "lll_r200_mpz_ref.json"), "w"), indent=2)
    print(rec)


def live_fixtures():
    """What the CPU tests once asked the reference for at run time, stored so that they run without it:
    ref_live.npz (GSO states after seeded op scripts, Householder dump digests along an HLLL-like call sequence, HLLL
    outputs on seeded bases), ref_islll.json (the reference's is_lll_reduced verdicts on a few bases),
    latticegen_r_12_200*.txt (a reference-written matrix and the reference's re-save of our writer's output) and
    strategies_default_*.json (an excerpt of strategies/default.json and digests of the whole parsed table)."""
    import json
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from fplll_b200 import io as fio
    import test_hh_oracle as T
    import test_oracle_golden as TG
    arrs = {}
    keys = ["n_known_rows", "n_known_cols", "n_source_rows", "row_expo", "gso_valid_cols", "init_row_size", "bf", "gf",
            "mu", "r", "b"]
    for seed, d, n, bits in TG.GSO_OPS_CASES:
        rng = np.random.default_rng(seed)
        b = rng.integers(-(1 << bits), 1 << bits, size=(d, n), dtype=np.int64)
        ops = H.random_op_script(rng, d, 40)
        s = O.RefSession(b)
        s.lines += H.ops_to_ref_script(ops)
        s.dump_state()
        rec = s.run()[1][0]
        arrs.update({"ops%d_%s" % (seed, k): rec[k] for k in keys})
    rng = np.random.default_rng(9)
    d = 10
    b = np.zeros((d, d + 1), np.int64)
    b[:, 0] = rng.integers(1, 1 << 40, size=d)
    b[np.arange(d), np.arange(d) + 1] = 1
    b[4] = 0
    s = O.RefSession(b)
    for t in range(3):
        s.cmd("update_row %d %d" % (t, t))
    s.dump_state()
    s.cmd("move_row 1 9")
    s.dump_state()
    for t, rec in enumerate(s.run()[1]):
        arrs.update({"ragged%d_%s" % (t, k): rec[k] for k in keys})
    for seed, d, n, bits in T.HH_SEQ_CASES:
        b, ops, rows_R = T.hh_call_sequence(seed, d, n, bits)
        tmp = O.tempfile.mkdtemp(prefix="hh_")
        mat, dump = os.path.join(tmp, "in.txt"), os.path.join(tmp, "d.bin")
        O.write_matrix(mat, b)
        script = ["load " + mat, "tolong", "hh 5"]
        for op in ops:
            script.append("hh_dump " + dump if op[0] == "dump" else
                          "hh_" + op[0] + " " + " ".join(str(int(x)) for x in op[1:]))
        O.run_ref("\n".join(script) + "\n")
        arrs["hh%d_digests" % seed] = np.array([H.hh_digest(r, rows_R) for r in O.read_hh_dumps(dump)])
    for seed, d, bits in T.HLLL_LIVE_CASES:
        rng = np.random.default_rng(seed)
        b = rng.integers(-(1 << bits), 1 << bits, size=(d, d), dtype=np.int64)
        pin, pout = os.path.join(TMP, "hlll_in.txt"), os.path.join(TMP, "hlll_out.txt")
        O.write_matrix(pin, b)
        o = O.run_ref("load %s\ntolong\nhlll_long 0.99 0.51 0.001 0.1\nsave_long %s\n" % (pin, pout))
        arrs["hlll%d_status" % seed] = np.int32(int(o.split("hlll_long status=")[1].split()[0]))
        arrs["hlll%d_out" % seed] = np.array(O.read_matrix(pout), dtype=np.int64)
    np.savez_compressed(os.path.join(HERE, "ref_live.npz"), **arrs)

    # is_lll_reduced<Z_NR<mpz_t>, FP_NR<mpfr_t>> (lll.cpp:226-258) at delta 0.99, eta 0.51
    u40, q60 = H.gold("u40_lll_long.npz"), H.gold("bkz_q60.npz")
    swapped = u40["b_out"].copy()
    swapped[[0, 1]] = swapped[[1, 0]]
    verdicts = {}
    for name, b in [("u40_b_in", u40["b_in"]), ("u40_b_out", u40["b_out"]), ("u40_b_out_rows_0_1_swapped", swapped),
                    ("q60_b_in", q60["b_in"]), ("q60_bkz30_default_b", q60["bkz30_default_b"])]:
        p = os.path.join(TMP, "islll.txt")
        O.write_matrix(p, b)
        verdicts[name] = int(O.run_ref("load %s\nislll 0.99 0.51\n" % p).split("islll ")[1].split()[0])
    json.dump(verdicts, open(os.path.join(HERE, "ref_islll.json"), "w"), indent=1)

    txt = O.latticegen(["r", 12, 200])
    open(os.path.join(HERE, "latticegen_r_12_200.txt"), "w").write(txt)
    p, q = os.path.join(TMP, "m.txt"), os.path.join(TMP, "m2.txt")
    fio.write_matrix(p, fio.read_matrix(txt))
    O.run_ref("load %s\nsave %s\n" % (p, q))
    open(os.path.join(HERE, "latticegen_r_12_200_resaved.txt"), "w").write(open(q).read())

    src = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "strategies", "default.json")
    table = fio.load_strategies_json(src)
    json.dump({str(bs): H.strategy_digest(v) for bs, v in sorted(table.items())},
              open(os.path.join(HERE, "strategies_default_digests.json"), "w"), indent=0)
    excerpt = [e for e in json.load(open(src)) if e["block_size"] in (0, 1, 2, 10, 20)]
    json.dump(excerpt, open(os.path.join(HERE, "strategies_default_excerpt.json"), "w"), separators=(",", ":"))


def size_class_inputs():
    """Seeded inputs of size_classes_ref.npz, which stores them for the tests: device LLL above 256 rows (d = 300, 12-bit entries;
    a d = 260 knapsack whose 40-60-bit column makes Babai round large X) and device HLLL with rows wider than 416
    columns (d = 30, n = 600)."""
    rng = np.random.default_rng(300)
    lll300 = rng.integers(-(1 << 12), 1 << 12, size=(300, 301), dtype=np.int64)
    knap260 = np.zeros((260, 261), np.int64)
    knap260[:, 0] = rng.integers(1 << 40, 1 << 60, size=260)
    knap260[np.arange(260), np.arange(260) + 1] = 1
    # 30 random rows of 600 columns are nearly orthogonal already: mix them so that HLLL has to work
    hlll600 = rng.integers(-64, 65, size=(30, 30)) @ rng.integers(-(1 << 10), 1 << 10, size=(30, 600))
    return dict(lll300=lll300, knap260=knap260, hlll600=hlll600)


def _narrow(a):
    """the smallest integer type that holds a exactly (keeps the fixture small; readers widen to int64)."""
    for t in (np.int16, np.int32):
        if np.abs(a).max() <= np.iinfo(t).max:
            return a.astype(t)
    return a


def size_class_fixtures():
    """tests/golden/size_classes_ref.npz (python tests/golden/make_golden.py --sizes, a few seconds): the reference's
    LLLReduction over MatGSO<long,double> with GSO_ROW_EXPO (ref_probe lll_long) and HLLLReduction<long,double>
    (hlll_long) on size_class_inputs(): input, output basis, status and, for LLL, the swap count."""
    pack = {}
    for tag, b in size_class_inputs().items():
        inp, outp = os.path.join(TMP, "size_%s_in.txt" % tag), os.path.join(TMP, "size_%s_out.txt" % tag)
        O.write_matrix(inp, b)
        cmd = "hlll_long 0.99 0.51 0.001 0.1" if tag.startswith("hlll") else "lll_long 0.99 0.51"
        o = O.run_ref("load %s\ntolong\n%s\nsave_long %s\n" % (inp, cmd, outp), timeout=600)
        tok = dict(t.split("=") for t in o.split(cmd.split()[0] + " ")[1].split() if "=" in t)
        pack[tag + "_in"] = _narrow(b)
        pack[tag + "_out"] = _narrow(np.array(O.read_matrix(outp), dtype=np.int64))
        pack[tag + "_status"] = np.int32(tok["status"])
        if "swaps" in tok:
            pack[tag + "_swaps"] = np.int32(tok["swaps"])
        print(tag, o.strip(), flush=True)
    np.savez_compressed(os.path.join(HERE, "size_classes_ref.npz"), **pack)


def enum_size_inputs():
    """Bases of enum_size_classes.npz, all from the LLL-reduced r200 basis (r200_lll_update_gso.npz).  An unpruned walk of
    an 80-row block of it never reaches a leaf in reasonable time, so two 80-row bases get a planted short vector: rows
    [120, 200) with every row but the first multiplied by 5 (b_0 is the shortest vector, about 8.7e5 nodes away), and the
    same rows with only the last one multiplied by 5 (the same for the dual, whose first vector is b*_79 / r_79)."""
    b = np.load(os.path.join(HERE, "r200_lll_update_gso.npz"))["b"]
    primal, dual = b[120:200].copy(), b[120:200].copy()
    primal[1:] *= 5
    dual[-1] *= 5
    return dict(r200=b, plant_primal=primal, plant_dual=dual)


# (name, basis, FIRST, LAST, FACTOR, pruning, ref_probe mode).  The radius is FACTOR * r(FIRST, FIRST), or FACTOR /
# r(LAST-1, LAST-1) for the dual; with these factors each of the reference's walks visits 2e5-1.5e6 nodes, well under
# a second.
ENUM_SIZE_CASES = [
    ("p80", "plant_primal", 0, 80, 1.01, None, "capture"),
    ("dual80", "plant_dual", 0, 80, 1.01, None, "capture_dual"),
    ("subsols80", "plant_primal", 0, 80, 1.01, None, "capture_subsols"),
    ("p100", "r200", 100, 200, 0.01, "strategy100", "capture"),
    ("p160", "r200", 40, 200, 1e-4, "linear", "capture"),
]


def enum_size_pruning(kind, d):
    """strategy100: the beta = 100 coefficients of strategies/default.json for the GH factor 1.0; linear: (d - i) / d."""
    if kind == "strategy100":
        z = np.load(os.path.join(os.path.dirname(os.path.dirname(HERE)), "fplll_b200", "data", "strategies_default.npz"))
        ghf = z["ghf_100"]
        return np.ascontiguousarray(z["coef_100"][int(np.argmin(np.abs(ghf - 1.0)))], np.float64)
    return (d - np.arange(d)) / float(d)


def enum_size_fixtures():
    """tests/golden/enum_size_classes.npz (python tests/golden/make_golden.py --enum-sizes, about a second): the reference's
    own enumerator above 64 dimensions through the capture hook (what the plugin API hands an external enumerator, then
    the internal enumerator runs) on ENUM_SIZE_CASES: the hook's mut / rdiag / pruning / radius, and the reference's
    per-level nodes, best vector and, for sub-solutions, the per-level best partial vectors."""
    bases = enum_size_inputs()
    out = os.path.join(TMP, "enum_size_fixture.bin")
    if os.path.exists(out):
        os.remove(out)
    script = []
    for name, base, first, last, factor, prune, mode in ENUM_SIZE_CASES:
        mat = os.path.join(TMP, "enum_size_%s.txt" % base)
        O.write_matrix(mat, bases[base])
        pf = "-"
        if prune:
            pf = os.path.join(TMP, "enum_size_%s.prune" % name)
            open(pf, "w").write(" ".join(repr(float(c)) for c in enum_size_pruning(prune, last - first)))
        script.append("load %s\ntolong\ngso l 2\nupdate_gso\nenum %d %d %r %s %s %s\n" % (mat, first, last, factor, pf,
                                                                                         out, mode))
    print(O.run_ref("".join(script), timeout=600))
    recs = O.read_enum_records(out)
    arrs = {}
    for (name, *_), r in zip(ENUM_SIZE_CASES, recs):
        arrs.update({name + "_mut": r["mut"], name + "_rdiag": r["rdiag"], name + "_pruning": r["pruning"],
                     name + "_maxdist": np.float64(r["maxdist"]), name + "_normexp": np.int64(r["normexp"]),
                     name + "_found": np.int32(r["found"]), name + "_best": np.float64(r["best"]),
                     name + "_sol": r["sol"], name + "_nodes": r["nodes"]})
        if r["subsols"]:
            arrs[name + "_subdist"] = r["subdist"]
            arrs[name + "_subsol"] = r["subsol"]
        print(name, "d", len(r["rdiag"]), "found", r["found"], "nodes", int(r["nodes"].sum()), flush=True)
    np.savez_compressed(os.path.join(HERE, "enum_size_classes.npz"), **arrs)


# (seed, d, bits, calls) of lll_ranged_ref.npz: full state dumps after every call at d <= 64, digests at d = 300
RANGED_CASES = [(11, 20, 10, 14), (12, 40, 12, 12), (13, 300, 12, 8)]


def ranged_fixtures():
    """tests/golden/lll_ranged_ref.npz (python tests/golden/make_golden.py --ranged): the reference's
    LLLReduction<Z_NR<long>, FP_NR<double>>::lll(kappa_min, kappa_start, kappa_end, size_reduction_start) and
    size_reduction on one MatGSO<long, double> object (GSO_ROW_EXPO) driven through helpers.ranged_call_script.  Per case:
    the input, the script, per call (ok, status, swaps, final_kappa, zeros) and a digest of the state (helpers.gso_digest);
    at d <= 64 also the state after every call (entries the reference leaves undefined are zeroed), at d = 300 the final
    basis."""
    import json
    pack = {}
    for case, (seed, d, bits, calls) in enumerate(RANGED_CASES):
        b = H.ranged_inputs(seed, d, bits)
        ops = H.ranged_call_script(np.random.default_rng(seed), d, calls)
        s = O.RefSession(b)
        for op in ops:
            s.lines += H.ranged_ref_lines(op)
            if op[0] in ("lll", "sr"):
                s.dump_state()
        out, recs = s.run()
        res = [[int(t.split("=")[1]) for t in line.split()[1:]] for line in out.splitlines()
               if line.startswith(("lll_range ", "size_reduction "))]
        assert len(res) == len(recs) == sum(op[0] in ("lll", "sr") for op in ops)
        p = "c%d_" % case
        pack[p + "b"] = _narrow(b)
        pack[p + "ops_json"] = np.frombuffer(json.dumps(ops).encode(), dtype=np.uint8)
        pack[p + "res"] = np.array(res, np.int32)
        pack[p + "digest"] = np.array([H.gso_digest(r) for r in recs])
        if d <= 64:
            for key in ["n_known_rows", "n_known_cols", "n_source_rows"]:
                pack[p + "s_" + key] = np.array([r[key] for r in recs], np.int32)
            for key in ["row_expo", "gso_valid_cols", "init_row_size", "b", "bf", "gf", "mu", "r"]:
                arrs = []
                for r in recs:
                    a = r[key].copy()
                    if key in ("mu", "r", "gf"):
                        keep = np.zeros(a.shape, bool)
                        for i in range(r["n_known_rows"]):
                            v = int(r["gso_valid_cols"][i])
                            keep[i, : {"mu": min(v, i), "r": v, "gf": i + 1}[key]] = True
                        a[~keep] = 0.0
                    arrs.append(a)
                pack[p + "s_" + key] = _narrow(np.array(arrs)) if key == "b" else np.array(arrs)
        else:
            pack[p + "b_out"] = _narrow(recs[-1]["b"])
        print("case", case, "d", d, "calls", len(res), "results", res, flush=True)
    np.savez_compressed(os.path.join(HERE, "lll_ranged_ref.npz"), **pack)


if __name__ == "__main__":
    if "--sizes" in sys.argv:
        size_class_fixtures()
    elif "--ranged" in sys.argv:
        ranged_fixtures()
    elif "--enum-sizes" in sys.argv:
        enum_size_fixtures()
    elif "--live" in sys.argv:
        live_fixtures()
    elif "--config2" in sys.argv:
        config2_mpz_reference()
    elif "--dual" in sys.argv:
        enum_dual_subsol_fixtures()
    elif "--configs" in sys.argv:
        config_size_fixtures()
    else:
        main()
