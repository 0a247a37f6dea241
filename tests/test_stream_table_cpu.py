"""CPU test of the host / device shared logic of the TMA streaming update kernel (fplll_b200/csrc/gso_stream.cuh): the
chunk-descriptor table every CTA builds must be exactly the sequence the consumer's loop nest waits for — b_i, then per
panel: bf chunks, mu rectangle chunks, the two halves of the diagonal tile — with the coordinates of the panel-packed
layout (gso_layout.cuh), and its byte total must be the row update's algorithmic bytes plus the documented slack (upper
halves of the first tile half, rows rounded to 2).  A mismatch here is a deadlock or silent garbage on the GPU."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "stream_table_check.cu")
EXE = os.path.join(ROOT, "tests", "_build", "stream_table_check")
SM_BF_FULL, SM_BF_PART, SM_MU_FULL, SM_MU_PART, SM_MU_B, SM_BROW = 0, 1, 2, 3, 4, 5
COLS = 16


@pytest.fixture(scope="module")
def exe():
    if not shutil.which("nvcc"):
        pytest.skip("nvcc not available")
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    deps = [SRC] + [os.path.join(ROOT, "fplll_b200", "csrc", f) for f in ("gso_stream.cuh", "tma.cuh", "gso_warp.cuh", "gso_layout.cuh")]
    if not os.path.exists(EXE) or any(os.path.getmtime(p) > os.path.getmtime(EXE) for p in deps):
        subprocess.check_call(["nvcc", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-o", EXE, SRC])
    return EXE


def table(exe, d, n, i, last_j):
    out = subprocess.run([exe, str(d), str(n), str(i), str(last_j)], capture_output=True, text=True, check=True).stdout
    lines = out.strip().splitlines()
    hdr = dict(t.split("=") for t in lines[0].split()[1:])
    rows = [tuple(int(x) for x in ln.split()) for ln in lines[1:]]
    return {k: int(v) for k, v in hdr.items()}, rows


def mu_panel_base(p):
    return 512 * p * (p + 1)


def expected(d, n, i, last_j):
    """The consumer's loop nest (stream_consumer / stream_panel), restated independently."""
    ldb = (n + 1) & ~1
    jl = min(last_j, i - 1)
    P = (jl >> 5) + 1 if jl >= 0 else 0
    rows_last = (((jl & 31) + 1 + 1) & ~1) if jl >= 0 else 32
    seq = [(SM_BROW, ldb * 8, 0, 0)]
    for p in range(P):
        part = (p == P - 1) and rows_last < 32
        rows = rows_last if part else 32
        for c0 in range(0, n, COLS):
            seq.append((SM_BF_PART if part else SM_BF_FULL, rows * COLS * 8, c0, p))
        col = mu_panel_base(p) // 32
        for c0 in range(0, 32 * p, COLS):
            seq.append((SM_MU_PART if part else SM_MU_FULL, rows * COLS * 8, col + c0, 0))
        seq.append((SM_MU_PART if part else SM_MU_FULL, rows * COLS * 8, col + 32 * p, 0))
        tile_cols = min(32, jl - 32 * p + 1)
        if tile_cols > 16:
            if part:
                seq.append((SM_MU_PART, rows * COLS * 8, col + 32 * p + 16, 0))
            else:
                seq.append((SM_MU_B, 16 * 16 * 8, col + 32 * p + 16, 16))
    return seq


@pytest.mark.parametrize("d,n,i,last_j", [(200, 201, 199, 199), (200, 201, 199, 150), (200, 201, 64, 64), (200, 201, 33, 33),
                                          (200, 201, 32, 32), (200, 201, 17, 17), (200, 201, 1, 1), (96, 96, 95, 95),
                                          (70, 75, 69, 62), (400, 400, 399, 399), (40, 40, 39, 39)])
def test_chunk_table_is_the_consumers_sequence(exe, d, n, i, last_j):
    hdr, rows = table(exe, d, n, i, last_j)
    exp = expected(d, n, i, last_j)
    assert hdr["NC"] == len(rows) == len(exp)
    for (e, mp, by, c1, c2), x in zip(rows, exp):
        assert (mp, by, c1, c2) == x, (e, (mp, by, c1, c2), x)
    # every copy is a multiple of 16 bytes and fits a stage
    assert all(r[2] % 16 == 0 and 0 < r[2] <= COLS * 32 * 8 for r in rows)


def test_streamed_bytes_against_the_algorithmic_bytes(exe):
    """update_gso_row(199) at n = 201 with the Gram row invalid: 8 [(i+1) n + i (i-1) / 2 + 4 (i+1)] = 485 608 algorithmic
    bytes (SURVEY §8 a2).  The stream fetches bf rows 0..198 and mu(j, k < j) plus, per full panel, the part of the first
    16 tile columns above the diagonal and the diagonal itself; the measured DRAM traffic of the kernel is 1.03x."""
    d, n, i = 200, 201, 199
    _, rows = table(exe, d, n, i, i)
    # OOB columns of the last bf chunk of a panel (n = 201 = 12 * 16 + 9) are zero-filled, not fetched
    fetched = 0
    for e, mp, by, c1, c2 in rows:
        if mp in (SM_BF_FULL, SM_BF_PART):
            cols = min(COLS, n - c1)
            fetched += by // COLS * cols
        else:
            fetched += by
    alg = 8 * ((i + 1) * n + i * (i - 1) // 2 + 4 * (i + 1))
    read_alg = 8 * (i * n + i * (i - 1) // 2)  # what of the algorithmic bytes is READ from bf and mu (rows j < i)
    assert read_alg <= fetched <= 1.06 * read_alg, (fetched, read_alg, alg)
