"""Static SASS evidence of the hot kernels: per-kernel opcode histogram + a few lines around the instructions that matter
(UTMALDG / UBLKCP / SYNCS = TMA + mbarrier, DMMA = fp64 tensor core, ATOMG / REDG .SYS = peer atomics).
usage: python tools/sass_excerpts.py > sass_excerpts.txt   (needs cuobjdump; no GPU)"""
import collections
import re
import subprocess

WANT = ["LDG", "LD", "LDS", "STS", "STG", "DMUL", "DADD", "DFMA", "DMMA", "SHFL", "UTMALDG", "UBLKCP", "UBLKPF", "SYNCS",
        "LDGSTS", "ATOM", "ATOMG", "RED", "REDG", "BAR", "IMAD", "BRA"]
KERNELS = [("fplll_b200/lib/libb200gso.so", "12k_update_rowE", r"LDG|DMUL|DADD", 8),
           ("fplll_b200/lib/libb200gso.so", "k_gram_tiles", r"DMMA", 6),
           ("fplll_b200/lib/libb200gso.so", "k_lll_ctaILi8", None, 0),
           ("fplll_b200/lib/libb200hh.so", "hk_update_R_x32", r"UTMALDG|SYNCS", 8),
           ("fplll_b200/lib/libb200hh.so", "hk_update_RILi14", r"DADD", 3),
           ("fplll_b200/lib/libb200enum.so", "k_enumILi64ELb1", r"ATOM|RED", 6)]


def functions(lib):
    text = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for ln in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur:
            funcs[cur].append(ln)
    return funcs


def main():
    for lib, pat, ex, nex in KERNELS:
        for name, lines in functions(lib).items():
            if pat not in name:
                continue
            c = collections.Counter()
            for ln in lines:
                m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", ln)
                if m:
                    c[m.group(1).split(".")[0]] += 1
            print("%s :: %s" % (lib.split("/")[-1], name[:110]))
            print("   %d SASS instructions; " % sum(c.values()) + ", ".join("%s %d" % (k, c[k]) for k in WANT if c[k]))
            if ex:
                for ln in [l.strip() for l in lines if re.search(ex, l)][:nex]:
                    print("      " + re.sub(r"\s+/\* 0x[0-9a-f]+ \*/", "", ln)[:150])
            print()


if __name__ == "__main__":
    main()
