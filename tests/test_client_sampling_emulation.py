"""The device's secret-key and error sampling maps (csrc/sampling.cuh over csrc/drbg.cuh), host-compiled, against the
restatement of the reference's randomizeTernary / randomizeCenteredBinomialDistribution (oracle/client_oracle.py); the
restatement pinned on fixed seeds and checked for its distribution."""
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import client_oracle as co

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEEDS = [bytes(range(32)), bytes(32), bytes.fromhex("69a09f6bf5dda15cd4af29e14cf5e0cddd7d07ac39bba587f8bc331104f9c448")]


@pytest.fixture(scope="module")
def emulator():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = tempfile.mkdtemp(prefix="sampling_emulate_")
    binary = os.path.join(out, "sampling_emulate")
    subprocess.check_call([nvcc, "-O1", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", binary,
                           os.path.join(ROOT, "tests", "emu", "sampling_emulate.cu")])
    yield binary
    shutil.rmtree(out, ignore_errors=True)


def _run(binary, *args):
    out = subprocess.run([binary, *map(str, args)], capture_output=True, text=True, check=True).stdout.split()
    return [int(v) for v in out]


@pytest.mark.parametrize("seed", SEEDS)
def test_ternary_map_matches_the_restatement_across_segment_ends(emulator, seed):
    # 12-byte coefficients: coefficient 341 straddles the first 4096-byte segment end, 682 the second
    count = 1100
    expected = [v + 1 for v in co.ternary_values(seed, count)]
    assert _run(emulator, seed.hex(), "ternary", 0, count) == expected
    assert _run(emulator, seed.hex(), "ternary", 335, 12) == expected[335:347]


@pytest.mark.parametrize("sigma", [co.STD_DEV_32, co.STD_DEV_64, 20.0])
@pytest.mark.parametrize("seed", SEEDS[:2])
def test_cbd_map_matches_the_restatement(emulator, seed, sigma):
    # 16 and 32 bytes per coefficient at stdDev32 / stdDev64; sigma 20 gives 26 words = 208 bytes, which straddle
    _, words, _ = co.cbd_shape(sigma)
    count = 3 * 4096 // (8 * words) + 7
    expected = co.cbd_values(seed, count, sigma)
    assert _run(emulator, seed.hex(), "cbd", sigma, 0, count) == expected
    assert _run(emulator, seed.hex(), "cbd", sigma, count - 5, 5) == expected[-5:]


def test_cbd_shapes():
    assert co.cbd_shape(co.STD_DEV_32) == (21, 2, (1 << 21) - 1)
    assert co.cbd_shape(co.STD_DEV_64) == (82, 4, (1 << 18) - 1)
    assert co.cbd_shape(8.0) == (128, 4, (1 << 64) - 1)


def test_restatement_pinned_on_fixed_seeds():
    assert co.ternary_values(bytes(range(32)), 16) == TERNARY_PIN
    assert co.cbd_values(bytes(range(32)), 16) == CBD32_PIN
    assert co.cbd_values(bytes(range(32)), 16, co.STD_DEV_64) == CBD64_PIN


def test_ternary_frequencies():
    values = np.array(co.ternary_values(b"\x07" * 32, 30000))
    for v in (-1, 0, 1):
        assert abs(np.mean(values == v) - 1 / 3) < 0.02


@pytest.mark.parametrize("sigma", [co.STD_DEV_32, co.STD_DEV_64])
def test_cbd_mean_and_variance(sigma):
    k, _, _ = co.cbd_shape(sigma)
    values = np.array(co.cbd_values(b"\x09" * 32, 20000, sigma), dtype=np.float64)
    assert abs(values.mean()) < 0.15
    assert abs(values.var() / (k / 2) - 1) < 0.08  # k trials a side: variance k / 2
    assert np.abs(values).max() <= k


# the first 16 coefficients of NistAes128Ctr(seed: 00 01 .. 1f) through each map (ternary values after the "- 1")
TERNARY_PIN = [0, 0, 1, 1, -1, 1, -1, 1, 1, -1, 1, 0, -1, -1, 0, 0]
CBD32_PIN = [4, -2, -3, -1, -1, 2, -4, -4, 5, -1, -1, 4, -8, 2, -4, -1]
CBD64_PIN = [3, -2, 5, -6, -7, -3, 2, 12, -5, -1, -5, 0, -4, 4, 10, -8]
