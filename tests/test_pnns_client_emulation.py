"""The PNNS client's device helpers (csrc/process_db.cuh: the float front end, the .denseRow / .denseColumn maps and the
plaintext CRT), host-compiled with FMA contraction off, against the restatement of the reference (tests/pnns_client_ref.py).
Rows where a contracted or reordered sum of squares changes the rounded integer are included and shown to discriminate,
so a build that contracts or reorders fails here."""
import os
import shutil
import subprocess
import tempfile
import types

import numpy as np
import pytest

from oracle import pnns_oracle as opn

import pnns_client_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emulator():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = tempfile.mkdtemp(prefix="pnns_client_emulate_")
    binary = os.path.join(out, "pnns_client_emulate")
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "-Xcompiler", "-ffp-contract=off",
                           "-o", binary, os.path.join(ROOT, "tests", "emu", "pnns_client_emulate.cu")])
    yield binary
    shutil.rmtree(out, ignore_errors=True)


def _run(binary, text):
    return subprocess.run([binary], input=text, capture_output=True, text=True, check=True).stdout.split("\n")[:-1]


def normalize(binary, vectors, s):
    v = np.ascontiguousarray(vectors, dtype=np.float32)
    text = f"norm {s} {v.shape[0]} {v.shape[1]}\n" + " ".join(f"{b:x}" for b in v.view(np.uint32).ravel())
    out = _run(binary, text)
    return None if "bad" in out else np.array([int(x) for x in out], dtype=np.int64).reshape(v.shape)


def sum_variants(vectors, s):
    """The rounded values with the sum of squares contracted into FMAs, and summed right to left."""
    v = np.asarray(vectors, dtype=np.float32)
    fma = np.zeros(v.shape[0], dtype=np.float32)
    rev = np.zeros(v.shape[0], dtype=np.float32)
    for k in range(v.shape[1]):
        fma = (fma.astype(np.float64) + v[:, k].astype(np.float64) ** 2).astype(np.float32)   # one rounding
        rev = (rev + v[:, -1 - k] * v[:, -1 - k]).astype(np.float32)
    out = []
    for total in (fma, rev):
        norm = np.sqrt(total).astype(np.float32)
        q = ((v * np.float32(s)).astype(np.float32) / norm[:, None]).astype(np.float32).astype(np.float64)
        out.append((np.floor(np.abs(q) + 0.5) * np.sign(q)).astype(np.int64))
    return out


def test_ties_round_away_from_zero(emulator):
    rows = [[1, 1, 1, 1], [-1, -1, -1, -1], [1, -1, 1, -1], [-3, 3, 3, -3]]
    got = normalize(emulator, rows, 101)                       # s / 2 = 50.5
    assert got.tolist() == ref.normalized_scaled_and_rounded(rows, 101)
    assert got[0].tolist() == [51] * 4 and got[1].tolist() == [-51] * 4


def test_zero_subnormal_and_large_rows(emulator):
    rows = np.array([[0, 0, 0, 0], [1e-40, 2e-40, 0, -3e-41], [1e-30, 2e-30, 3e-30, 4e-30], [1e20, 1, -2, 3],
                     [3e18, -4e18, 0, 1e18]], dtype=np.float32)
    assert normalize(emulator, rows, 1000).tolist() == ref.normalized_scaled_and_rounded(rows.tolist(), 1000)


def test_traps(emulator):
    for bad in (np.inf, -np.inf, np.nan):
        assert normalize(emulator, [[1.0, bad]], 10) is None
    assert normalize(emulator, [[1.0, 0.0]], 2 ** 63) is None   # Float(2^63) leaves Int64


@pytest.mark.parametrize("cols", [512, 1024])
def test_random_rows(emulator, cols):
    rng = np.random.default_rng(cols)
    v = (rng.standard_normal((64, cols)) * rng.uniform(0.01, 100, (64, 1))).astype(np.float32)
    for s in (169, 65525, 1 << 20):
        assert np.array_equal(normalize(emulator, v, s), ref.normalized_scaled_and_rounded_array(v, s))


def test_contracted_or_reordered_sums_are_caught(emulator):
    s, cols = 1 << 22, 1024
    rng = np.random.default_rng(11)
    v = rng.standard_normal((3000, cols)).astype(np.float32)
    exact = ref.normalized_scaled_and_rounded_array(v, s)
    fma, rev = sum_variants(v, s)
    fma_rows = np.nonzero(np.any(fma != exact, axis=1))[0]
    rev_rows = np.nonzero(np.any(rev != exact, axis=1))[0]
    assert len(fma_rows) and len(rev_rows)                     # the rows discriminate
    picked = np.unique(np.concatenate([fma_rows[:8], rev_rows[:8]]))
    assert np.array_equal(normalize(emulator, v[picked], s), exact[picked])
    assert np.any(fma[picked] != exact[picked]) and np.any(rev[picked] != exact[picked])


def _dense_row_labels(monkeypatch, rows, cols, n):
    """The oracle's .denseRow packing of values labelled 1 .. rows * cols, before encoding (0 = padding)."""
    monkeypatch.setattr(opn, "encode_simd", lambda ctx, values: list(values))
    ctx = types.SimpleNamespace(n=n, t=1 << 62)
    return opn.dense_row_plaintexts(ctx, rows, cols, list(range(1, rows * cols + 1)))


@pytest.mark.parametrize("n,rows,cols", [(16, 1, 3), (16, 3, 4), (16, 5, 3), (64, 7, 5), (64, 32, 16), (64, 9, 32),
                                         (512, 17, 32), (1024, 3, 300), (8192, 16, 512)])
def test_dense_row_map(emulator, monkeypatch, n, rows, cols):
    expected = _dense_row_labels(monkeypatch, rows, cols, n)
    out = [int(x) for x in _run(emulator, f"dense_row {rows} {cols} {n.bit_length() - 1}")]
    assert len(out) == len(expected) * n
    assert [x + 1 for x in out] == [int(v) for p in expected for v in p]


@pytest.mark.parametrize("n,rows,cols", [(16, 1, 3), (16, 3, 4), (16, 8, 3), (16, 9, 2), (16, 20, 3), (64, 65, 1),
                                         (64, 32, 16), (64, 192, 1), (8192, 2000, 16), (8192, 100000, 3)])
def test_dense_column_map(emulator, n, rows, cols):
    out = _run(emulator, f"dense_column {rows} {cols} {n.bit_length() - 1}")
    count = int(out[0])
    labels = [[p * n + j for j in range(n)] for p in range(count)]
    ctx = types.SimpleNamespace(n=n)
    expected = opn.unpack_dense_column(ctx, labels, rows, cols)
    got = [int(a) * n + int(b) for a, b in (line.split() for line in out[1:])]
    assert got == expected


@pytest.mark.parametrize("moduli", [[65537], [65537, 114689], [40961, 65537, 114689]])
def test_crt(emulator, moduli):
    rng = np.random.default_rng(len(moduli))
    t = int(np.prod(moduli, dtype=object))
    values = [int(x) for x in rng.integers(-(t // 2), (t - 1) // 2, size=200)] + [-(t // 2), (t - 1) // 2, 0, -1, 1]
    s = 169 if len(moduli) == 1 else 65525
    text = f"crt {len(moduli)} {' '.join(map(str, moduli))} {s} {len(values)}\n" + \
        "\n".join(" ".join(str(v % m) for m in moduli) for v in values)
    out = [line.split() for line in _run(emulator, text)]
    residues = [[v % m for v in values] for m in moduli]
    composed = [ref.remainder_to_centered(x, t) for x in ref.crt_compose(residues, moduli)]
    assert composed == values
    assert [int(a) for a, _ in out] == values
    expected = ref.distances_from_signed([values], s)[0]
    assert [int(b, 16) for _, b in out] == expected.view(np.uint32).tolist()
