"""Compares the SASS of two builds of the same object, kernel by kernel (cuobjdump -sass), ignoring instruction
addresses and encodings; template instantiations are matched by the name with the anonymous-namespace hash removed
and an optional rename applied.  Used to show that adding a template parameter left the existing instantiations'
instructions unchanged:
    python tools/sass_diff.py OLD.o NEW.o [--map 'ILi4EEE=ILi4ELb0EEE' ...] [--only k_lll k_update_row ...]
--param-shift OFF:DELTA compares an old kernel-parameter load c[0x0][X] with X >= OFF as c[0x0][X + DELTA]: appending
fields to a struct passed by value moves the parameters behind it, and nothing else.
Prints one line per kernel of OLD: identical, or the number of differing instruction lines."""
import argparse
import re
import subprocess


def kernels(obj):
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, name, body = {}, None, []
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            if name:
                funcs[name] = body
            name, body = re.sub(r"_GLOBAL__N__[0-9a-f]+_", "_GLOBAL__N__", m.group(1)), []
            continue
        if name is None:
            continue
        ins = re.sub(r"/\*[0-9a-f]{4,}\*/", "", line)  # address
        ins = re.sub(r"/\* 0x[0-9a-f]+ \*/", "", ins).strip()  # encoding
        if ins and not ins.startswith(".") and ins != "}" and ins != "{":
            body.append(ins)
    if name:
        funcs[name] = body
    return funcs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--map", nargs="*", default=[], help="OLD=NEW substrings applied to the old kernel names")
    ap.add_argument("--only", nargs="*", default=[], help="compare only kernels whose name contains one of these")
    ap.add_argument("--param-shift", default=None, help="OFF:DELTA (hex or decimal bytes)")
    a = ap.parse_args()
    shift = None
    if a.param_shift:
        off, delta = (int(t, 0) for t in a.param_shift.split(":"))

        def shift(ins):
            return re.sub(r"c\[0x0\]\[0x([0-9a-f]+)\]",
                          lambda m: "c[0x0][%s]" % hex(int(m.group(1), 16) + (delta if int(m.group(1), 16) >= off else 0)),
                          ins)
    old, new = kernels(a.old), kernels(a.new)
    bad = 0
    for name, body in sorted(old.items()):
        if a.only and not any(s in name for s in a.only):
            continue
        target = name
        for m in a.map:
            o, n = m.split("=")
            target = target.replace(o, n)
        if target not in new:
            print("MISSING %s" % target)
            bad += 1
            continue
        nb = new[target]
        if shift:
            body = [shift(x) for x in body]
        diff = sum(1 for x, y in zip(body, nb) if x != y) + abs(len(body) - len(nb))
        print("%-9s %s (%d instructions)" % ("identical" if diff == 0 else "DIFF %d" % diff, name, len(body)))
        bad += diff != 0
    raise SystemExit(1 if bad else 0)


if __name__ == "__main__":
    main()
