"""CPU checks of the N = 8192 resident twiddle image (csrc/ntt_fast.cuh, resident_twiddles): which entries it keeps,
that zeta = psi^(+-N/2) recovers the ones it drops, that it fits a CTA's shared memory next to the two row buffers,
that the image context.cu builds puts each entry where the kernels read it, and that those reads are bank-conflict
free.  tests/test_ntt_emulation.py replays the kernels' pass functions at N = 8192, with the entries they keep and the
zeta step."""
import os
import shutil
import subprocess

import pytest

from oracle import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "swift-homomorphic-encryption_b200", "csrc")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
LOGN = 13
N, T = 1 << LOGN, (1 << LOGN) // 16
SLOTS = 11
FWD_K = [k if k < 7 else 7 + 2 * (k - 7) for k in range(SLOTS)]  # fwd_image_k
INV_K = [2 * k if k < 4 else k + 4 for k in range(SLOTS)]        # inv_image_k


def test_slots_keep_all_but_the_odd_groups_of_the_zeta_stage():
    # forward stage j owns transposed entries 2^j - 1 + grp (grp < 2^j); stage 3 has the N/2 twiddles
    assert sorted(FWD_K) == [k for k in range(15) if not (k >= 7 and (k - 7) % 2)]
    # inverse stage J owns 16 - (16 >> J) + grp (grp < 2^(3-J)); stage 0 has the N/2 twiddles
    assert sorted(INV_K) == [k for k in range(15) if not (k < 8 and k % 2)]


def test_shared_memory_budget():
    rows = 2 * N * 8
    image = (T + SLOTS * T) * 16
    assert image == 96 * 1024
    assert rows + image + 3 * 8 == 229400 <= 232448       # the opt-in limit of one CTA on sm_90
    assert rows + (T + 15 * T) * 16 + 3 * 8 > 232448      # all 15 entries a thread would not fit


@pytest.mark.parametrize("bits", [25, 30, 50, 55, 61, 62])
def test_zeta_recovers_the_odd_entries(bits):
    """tw[N/2 + i] = tw[N/2 + i - 1] tw[1] for odd i (tables in bit-reversed order: i and i - 1 differ by N/2 in the
    exponent of psi), forward and inverse"""
    p = orc.generate_primes([bits], False, N)[0]
    psi = next(r for r in (pow(g, (p - 1) // (2 * N), p) for g in range(2, 1000)) if pow(r, N, p) == p - 1)
    for root in (psi, pow(psi, -1, p)):
        w = [0] * N  # context.cu: tw[bitrev(i)] = psi^i
        for i in range(N):
            w[orc.reverse_bits(i, LOGN)] = pow(root, i, p)
        zeta = w[1]
        assert pow(zeta, 2, p) == p - 1  # a square root of -1: psi^(N/2)
        assert all(w[i] == w[i - 1] * zeta % p for i in range(N // 2 + 1, N, 2))


IMAGE_PROBE = r"""
#include <cstdio>
#include "ntt_fast.cuh"
int main() {
    using namespace hecuda::fast;
    for (int inv = 0; inv < 2; ++inv)
        for (int i = 0; i < image_entries(13); ++i) printf("%d\n", image_source(13, inv != 0, i));
    return 0;
}
"""


def _expected_source(inverse, i):
    """table index of image entry i, from the pass structure: the kernels read slot k' of thread tau at
    N/16 + k' T + tau, and slot k' holds transposed entry k = FWD_K[k'] / INV_K[k'] of that thread"""
    if i < T:
        return i
    kp, tau = i // T - 1, i % T
    if not inverse:
        k = FWD_K[kp]
        j = next(j for j in range(4) if (1 << j) - 1 <= k < (2 << j) - 1)  # forward stage j: 2^j groups
        return (1 << (LOGN - 4 + j)) + (tau << j) + k - ((1 << j) - 1)
    k = INV_K[kp]
    J = next(J for J in range(4) if 16 - (16 >> J) <= k < 16 - (16 >> (J + 1)))  # inverse stage J: 2^(3-J) groups
    return (1 << (LOGN - 1 - J)) + (tau << (3 - J)) + k - (16 - (16 >> J))


def test_image_layout_matches_the_kernels_reads(tmp_path):
    """image_source (what context.cu copies into the image) against the kernels' read order"""
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    src, exe = tmp_path / "probe.cu", tmp_path / "probe"
    src.write_text(IMAGE_PROBE)
    subprocess.check_call([NVCC, "-O1", "-std=c++17", "-Wno-deprecated-gpu-targets", "-I", CSRC, "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    entries = (1 + SLOTS) * T
    assert got == [_expected_source(False, i) for i in range(entries)] + [_expected_source(True, i) for i in range(entries)]
    for d in (0, 1):  # every table index at most once per direction
        assert len(set(got[d * entries:(d + 1) * entries])) == entries


@pytest.mark.parametrize("slot", range(SLOTS))
def test_image_reads_are_conflict_free(slot):
    """a warp reads slot k' of its 32 threads at words 2 (T + k' T + tau): 512 contiguous bytes, served per quarter
    warp (8 lanes x 16 bytes must hit 8 distinct 16-byte bank groups)"""
    for w0 in range(0, T, 8):
        groups = [(T + slot * T + tau) % 8 for tau in range(w0, w0 + 8)]
        assert len(set(groups)) == 8
