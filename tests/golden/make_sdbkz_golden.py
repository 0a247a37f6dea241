"""Regenerates tests/golden/bkz_sd_sld.npz (the SD-BKZ / slide-reduction and dual-enumeration fixtures) from the
UNMODIFIED reference (oracle/_ref, built from the reference sources by oracle/Makefile.ref).  Run in the build
container only, after the fixtures it reads (bkz_q60.npz, bkz_gm180.npz, r200_lll_update_gso.npz) exist:
    python tests/golden/make_sdbkz_golden.py [OUT.npz]
Inputs are existing fixtures or come from the reference's own latticegen; ~2 min of CPU."""
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


def sdbkz_fixtures(out_path=None):
    """SD-BKZ (BKZ_SD_VARIANT 0x100) and slide reduction (BKZ_SLD_RED 0x200) through the reference's own bkz_reduction,
    plus a full-size dual enumeration -> `out` (default tests/golden/bkz_sd_sld.npz)
      * unpruned runs on bkz_q60.npz:b_in (deterministic: the output basis is the known answer) and one SD-BKZ-40 loop on
        bkz_gm180.npz:b_in; default-strategy runs on the q60 basis (status and output, for quality gates);
      * dual SVP enumeration of block [140, 200) of the LLL-reduced r200 basis with the beta = 60 pruning vector of
        strategies/default.json at the radius svp_reduction sets (delta / r(199, 199)), through the capture hook: mu^T,
        rdiag, pruning, the reference's best dual vector, its distance and per-level nodes."""
    import json
    import time
    NO_LLL, MAX_LOOPS, BOUNDED_LLL, SD, SLD = 2, 4, 0x10, 0x100, 0x200
    pack = {}
    q60 = H.gold("bkz_q60.npz")["b_in"]
    gm = H.gold("bkz_gm180.npz")["b_in"]
    cases = [("sd20_none", q60, 20, SD | NO_LLL | MAX_LOOPS, 2, "none"),
             ("sld20_none", q60, 20, SLD | NO_LLL, 0, "none"),
             ("sld20_bounded_none", q60, 20, SLD | NO_LLL | BOUNDED_LLL, 0, "none"),
             ("sd30_default", q60, 30, SD | NO_LLL | MAX_LOOPS, 2, "default"),
             ("sld30_default", q60, 30, SLD | NO_LLL, 0, "default"),
             ("gm180_sd40_none", gm, 40, SD | NO_LLL | MAX_LOOPS, 1, "none")]
    for tag, b_in, bs, fl, ml, strat in cases:
        inp, outp = os.path.join(TMP, "sdbkz_%s_in.txt" % tag), os.path.join(TMP, "sdbkz_%s_out.txt" % tag)
        O.write_matrix(inp, b_in)
        t0 = time.time()
        o = O.run_ref("load %s\nbkz %d %d %d %s enumlib 1\nsave %s\n" % (inp, bs, fl, ml, strat, outp), timeout=1800)
        pack[tag + "_status"] = np.int32(int(o.split("bkz status=")[1].split()[0]))
        pack[tag + "_b"] = np.array(O.read_matrix(outp), dtype=np.int64)
        pack[tag + "_flags"] = np.int32(fl)
        print(tag, "status", int(pack[tag + "_status"]), "sec %.1f" % (time.time() - t0), flush=True)
    # dual enumeration, d = 60
    g = np.load(os.path.join(HERE, "r200_lll_update_gso.npz"))
    mat = os.path.join(TMP, "r200_red.txt")
    O.write_matrix(mat, g["b"])
    strat = json.load(open(os.path.join(O.REF_DIR, "strategies", "default.json")))
    pr60 = [e for e in strat if e["block_size"] == 60][0]["pruning_parameters"][15]
    prfile = os.path.join(TMP, "prune60.txt")
    open(prfile, "w").write(" ".join(repr(float(c)) for c in pr60[1]))
    out = os.path.join(TMP, "enum_dual60_fixture.bin")
    if os.path.exists(out):
        os.remove(out)
    t0 = time.time()
    O.run_ref("load %s\ntolong\ngso l 2\nupdate_gso\nenum 140 200 0.99 %s %s capture_dual\n" % (mat, prfile, out),
              timeout=1800)
    r = O.read_enum_records(out)[0]
    print("dual60 found", r["found"], "nodes", int(r["nodes"].sum()), "sec %.1f" % (time.time() - t0), flush=True)
    pack.update(dual60_mut=r["mut"], dual60_rdiag=r["rdiag"], dual60_pruning=r["pruning"],
                dual60_maxdist=np.float64(r["maxdist"]), dual60_normexp=np.int64(r["normexp"]),
                dual60_found=np.int32(r["found"]), dual60_best=np.float64(r["best"]), dual60_sol=r["sol"],
                dual60_nodes=r["nodes"])
    # d = 40: the last 40 rows of the same block (a block of their own), unpruned, radius delta / r(199, 199); the
    # oracle's shrinking walk (pinned to the reference's enumerator in tests/test_enum_oracle.py) gives the best vector
    mut40, rdiag40 = np.ascontiguousarray(r["mut"][20:, 20:]), np.ascontiguousarray(r["rdiag"][20:])
    R40 = 0.99 / float(rdiag40[-1])
    o40 = O.enum_svp_ex(mut40, rdiag40, None, R40, shrink=True, dual=True)
    pack.update(dual40_mut=mut40, dual40_rdiag=rdiag40, dual40_maxdist=np.float64(R40), dual40_best=np.float64(o40["best"]),
                dual40_sol=o40["sol"])
    # the oracle's fixed-radius walks at radii that keep them short (the device must visit exactly these nodes): d = 60
    # just outside the reference's best vector (5.9e7 nodes; the region of the full radius has billions)
    best60 = float(r["best"]) / 2.0 ** int(r["normexp"])
    for tag, mut, rdiag, prun, R in (("dual40", mut40, rdiag40, None, 0.5 * R40),
                                     ("dual60", r["mut"], r["rdiag"], r["pruning"], 1.02 * best60)):
        ref = O.enum_svp_ex(mut, rdiag, prun, R, shrink=False, dual=True)
        pack[tag + "_fixed_R"] = np.float64(R)
        pack[tag + "_fixed_nodes"] = ref["nodes"]
        print(tag, "fixed-radius oracle nodes", int(ref["nodes"].sum()), flush=True)
    np.savez_compressed(out_path or os.path.join(HERE, "bkz_sd_sld.npz"), **pack)


if __name__ == "__main__":
    sdbkz_fixtures(sys.argv[1] if len(sys.argv) > 1 else None)
