"""In-tree nvcc build of the CUDA extension (sm_90a, H100, only).  The .so stays in fplll_b200/lib/ (git-ignored,
travels to the GPU box with the snapshot)."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
# B200_LIB_DIR: build/load a variant (other -D flags) next to the default one; the default is what ships
LIBDIR = os.path.join(HERE, os.environ.get("B200_LIB_DIR", "lib"))
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + [ "-lineinfo", "-O3", "-std=c++17",
              # the reference build never contracts a*b+c (configure.ac:25: -O3, no -march): bit parity needs the same
              "--fmad=false", "-Xcompiler", "-fPIC", "-shared"]

TARGETS = {
    "libb200gso.so": ["gso_api.cu", "gso_lll_api.cu", "gso_lll_cta_api.cu"],
    "libb200enum.so": ["enum_api.cu"],
    "libb200bkz.so": ["gso_api.cu", "gso_lll_api.cu", "gso_lll_cta_api.cu", "enum_api.cu", "bkz_api.cu"],
    "libb200hh.so": ["hh_api.cu"],
}


def _deps(src, seen=None):
    """The unit's own quoted #include closure (csrc/*.cuh and include/*.h): an edit rebuilds only the units that see it."""
    import re
    seen = set() if seen is None else seen
    src = os.path.normpath(src)
    if src in seen or not os.path.exists(src):
        return seen
    seen.add(src)
    for inc in re.findall(r'^\s*#\s*include\s+"([^"]+)"', open(src).read(), flags=re.M):
        _deps(os.path.join(os.path.dirname(src), inc), seen)
    return seen


def _stale(out, srcs):
    if not os.path.exists(out):
        return True
    deps = set()
    for s in srcs:
        _deps(s, deps)
    return any(os.path.getmtime(p) > os.path.getmtime(out) for p in deps)


def build_all(force=False, verbose=False):
    """Each .cu is compiled ONCE to an object, all translation units in parallel (the LLL kernels — three Babai widths,
    fully unrolled — live in units of their own because they take minutes), then every library is linked from the objects
    it needs.  No --split-compile: its code generation is not reproducible from run to run."""
    from concurrent.futures import ThreadPoolExecutor
    objdir = os.path.join(LIBDIR, "obj")
    os.makedirs(objdir, exist_ok=True)
    # B200_NVCC_EXTRA: extra compile flags for experiments, e.g. -DB200_LLL_PROFILE (device-clock phase counters)
    cflags = [f for f in NVCC_FLAGS if f != "-shared"] + os.environ.get("B200_NVCC_EXTRA", "").split()
    units = sorted({u for srcs in TARGETS.values() for u in srcs})

    def compile_unit(u):
        src, obj = os.path.join(CSRC, u), os.path.join(objdir, u[:-3] + ".o")
        if force or _stale(obj, [src]):
            subprocess.check_call(["nvcc"] + cflags + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", obj, src])
        return obj

    with ThreadPoolExecutor(max_workers=len(units)) as ex:
        objs = dict(zip(units, ex.map(compile_unit, units)))
    built = []
    for name, srcs in TARGETS.items():
        out = os.path.join(LIBDIR, name)
        deps = [objs[u] for u in srcs]
        if force or not os.path.exists(out) or any(os.path.getmtime(o) > os.path.getmtime(out) for o in deps):
            cmd = ["nvcc", "-shared"] + ARCH + ["-o", out] + deps
            if name == "libb200enum.so" and os.environ.get("B200_WITH_NCCL"):
                cmd += ["-lnccl"]
            subprocess.check_call(cmd)
        built.append(out)
    return built


if __name__ == "__main__":
    import sys
    print("\n".join(build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)))
