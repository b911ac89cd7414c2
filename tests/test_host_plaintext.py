"""The plaintext side of the C++ mirror (host/HeScheme.hpp: encodeSimd / decodeSimd / addAssignCoeff / subAssignCoeff /
subCoeff): compiles and links on CPU; on a GPU its results match the reference restatement in tests/plaintext_ref.py."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "host_plaintext_test.cpp")
LIBDIR = os.path.join(ROOT, "swift-homomorphic-encryption_b200")


def build(tmp_path):
    out = str(tmp_path / "host_plaintext_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-o", out, SRC, "-L" + LIBDIR, "-lhecuda",
                           "-Wl,-rpath," + LIBDIR])
    return out


def test_host_plaintext_mirror_compiles_and_links(tmp_path):
    assert os.path.exists(os.path.join(LIBDIR, "libhecuda.so")), "build libhecuda.so first"
    build(tmp_path)


@pytest.mark.gpu
def test_host_plaintext_mirror_matches_reference(tmp_path):
    import plaintext_ref as ref

    exe = build(tmp_path)
    out = tmp_path / "out.bin"
    run = subprocess.run([exe, str(out)], capture_output=True, text=True)
    assert run.returncode == 0, run.stderr
    n, moduli, t = 4096, [134176769, 268369921, 268361729], 65537
    L = 2
    data = np.fromfile(out, dtype=np.uint64)
    ct, pt = data[: 2 * L * n].reshape(2, L, n), data[2 * L * n: 2 * L * n + n]
    rest = data[2 * L * n + n:].reshape(3, 2, L, n)
    for got, op in zip(rest, (ref.ADD, ref.SUB, ref.SUB_FROM)):
        assert np.array_equal(got, ref.plaintext_translate(moduli, t, ct, pt, op)), op
