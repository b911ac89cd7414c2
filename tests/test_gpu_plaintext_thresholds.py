"""GPU parity at the plaintext side's rounding and centring thresholds (tests/plaintext_thresholds.py builds the inputs).

A uniform plaintext coefficient puts a decision on its threshold with probability 1 / t, so a `>=` written as `>` in one
of these kernels passes every other parity test once t is more than a few thousand.  Here every plaintext holds each
constructed value at several positions, including 0 and N - 1, and the results are compared bit-exactly with the oracle:

  D1 translate  kernels.cuh translate_adjust        through addAssignCoeff / subAssignCoeff / subCoeff (host buffers and
                                                    the device-pointer entry point, 2 and 3 polynomials, one plaintext per
                                                    ciphertext and one shared) at every level, and through encryption
  D2 lift       innerprod.cu plaintext_lift_kernel  through plaintextToEval and encodeSimd(moduliCount: l) at every level,
                                                    and through MulPir database processing (host and device packing)
  D3 uncentre   plaintext.cu uncenter_kernel        through decodeSimd(moduliCount: l) of Eval plaintexts at every level

The matrix (plaintext_thresholds.CONTEXTS), each t with its own context:
  Bfv<UInt64>  t = 2 (N = 16), 97 (N = 16), 17 and 65537 (n_4096_logq_27_28_28), 4294828033 and 4294991873 (the
               NTT-friendly primes on either side of 2^32, where the reference's translate switches from one-word to
               double-width division), 33832961 and 2199023288321 (N = 8192 predefined sets; the latter is the 42-bit t
               of n_8192_logq_3x55_logt_42) and 2305843009213554689 (61 bits, under four 62-bit moduli)
  Bfv<UInt32>  t = 40961 and 65537 (either side of 2^16) at n_4096_logq_27_28_28, and 536813569 (29 bits) under four
               30-bit moduli
Bfv<UInt32> has no encryption or plaintextToEval entry point, and decodeSimd needs a SIMD t (not 2 or 17 at N = 4096):
those contexts reach the other decisions only."""
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda
from hecuda import pir
import plaintext_ref as ref
import plaintext_thresholds as pt
from oracle import client_oracle as co
from oracle import oracle as orc
from oracle import pnns_oracle as pn
from test_gpu_evk_wire import read_device

OPS = {ref.ADD: "addAssignCoeff", ref.SUB: "subAssignCoeff", ref.SUB_FROM: "subCoeff"}
U64 = [c for c in pt.CONTEXTS if c[4] == 64]
SIMD = [c for c in pt.CONTEXTS if pt.simd(c[1], c[3])]


def ids(cases):
    return [c[0] for c in cases]


def contexts(n, moduli, t, word_bits):
    g = hecuda.Context(n, moduli, t, scalar=np.uint32 if word_bits == 32 else np.uint64)
    return g, orc.Context(n, moduli, t, word_bits=word_bits), (hecuda.Bfv32 if word_bits == 32 else hecuda.Bfv)


def words(a, word_bits):
    return np.asarray(a, dtype=np.uint32 if word_bits == 32 else np.uint64)


def seed(i: int) -> bytes:
    return random.Random(i).randbytes(32)


def lift_plaintexts(n, t, rs):
    """(V, N) Coeff plaintexts holding every lift input (thr - 1, thr, thr + 1, 0, 1, t - 1) at 0, N - 1 and more."""
    return pt.threshold_polys(pt.lift_inputs(t), n, t, random.Random(rs))[0]


@pytest.mark.parametrize("name,n,moduli,t,word_bits", pt.CONTEXTS, ids=pt.IDS)
def test_context_is_accepted(name, n, moduli, t, word_bits):
    """Every t of the matrix, up to 61 bits under 62-bit moduli and 29 bits under 30-bit moduli, makes a context."""
    g, o, _ = contexts(n, moduli, t, word_bits)
    assert g.L == o.L == len(moduli) - 1
    assert g.supportsSimdEncoding == pt.simd(n, t)
    g.close()


# ------------------------------------------------------------------------------------------------------- D1 translate
def _device_translate(g, ct, plain, op):
    import torch

    batch, polys, l, _ = ct.shape
    lib, s = hecuda.load_library(), torch.cuda.current_stream().cuda_stream
    d_ct, d_pt = torch.from_numpy(ct.view(np.int64)).cuda(), torch.from_numpy(np.ascontiguousarray(plain).view(np.int64)).cuda()
    d_out = torch.empty_like(d_ct)
    count = plain.size // g.degree
    hecuda._check(lib.hecuda_bfv_plaintext_translate_device(g._h, d_ct.data_ptr(), polys, l, d_pt.data_ptr(), count, op,
                                                            d_out.data_ptr(), batch, s))
    torch.cuda.synchronize()
    return d_out.cpu().numpy().view(np.uint64)


def _translate(bfv, g, op, ct, plain):
    if op == ref.SUB_FROM:
        return bfv.subCoeff(g, plain, ct)
    return getattr(bfv, OPS[op])(g, ct, plain)


@pytest.mark.parametrize("name,n,moduli,t,word_bits", pt.CONTEXTS, ids=pt.IDS)
def test_translate_at_carry_threshold(name, n, moduli, t, word_bits):
    """Every m of translate_inputs at every level, for each op, per-ciphertext and shared plaintexts, 2 and 3
    polynomials; Bfv<UInt64> also through the device-pointer entry point."""
    g, o, bfv = contexts(n, moduli, t, word_bits)
    rng = random.Random(t ^ n)
    for l in range(o.L, 0, -1):
        ms = [m for m, _ in pt.translate_inputs(moduli, t, l)]
        plain, _ = pt.threshold_polys(ms, n, t, rng)
        batch = len(ms)
        for polys in (2, 3):
            ct = orc.fill_uniform(l * 7 + polys, moduli[:l], n, batch * polys * l).reshape(batch, polys, l, n)
            for op in OPS:
                per = np.stack([ref.plaintext_translate(moduli, t, ct[i], plain[i], op) for i in range(batch)])
                shared = np.stack([ref.plaintext_translate(moduli, t, ct[i], plain[0], op) for i in range(batch)])
                case = (l, polys, op)
                got = _translate(bfv, g, op, words(ct, word_bits), words(plain, word_bits))
                assert np.array_equal(got.astype(np.uint64), per), case
                got = _translate(bfv, g, op, words(ct, word_bits), words(plain[0], word_bits))
                assert np.array_equal(got.astype(np.uint64), shared), case
                if word_bits == 64:
                    assert np.array_equal(_device_translate(g, ct, plain, op), per), case + ("device",)
                    assert np.array_equal(_device_translate(g, ct, plain[:1], op), shared), case + ("device",)
    g.close()


@pytest.mark.parametrize("name,n,moduli,t,word_bits", U64, ids=ids(U64))
def test_encrypt_at_carry_threshold(name, n, moduli, t, word_bits):
    """Fresh encryptions of plaintexts holding every translate input of the top level equal the oracle's for the same
    seeds and decrypt back."""
    g, o, _ = contexts(n, moduli, t, word_bits)
    L = g.L
    ms = [m for m, _ in pt.translate_inputs(moduli, t, L)]
    plain, _ = pt.threshold_polys(ms, n, t, random.Random(t + 3))
    sk = hecuda.SecretKey.generate(g, seed(1))
    a = [seed(10 + i) for i in range(len(ms))]
    e = [seed(40 + i) for i in range(len(ms))]
    cts = hecuda.Bfv.encrypt(g, sk, plain, aSeeds=b"".join(a), errorSeeds=b"".join(e))
    for i in range(len(ms)):
        assert np.array_equal(cts[i], co.encrypt(n, moduli[:L], t, sk.poly, plain[i], a[i], e[i])), i
    assert np.array_equal(hecuda.Bfv.decrypt(g, cts, sk), plain)
    g.close()


# ------------------------------------------------------------------------------------------------------------ D2 lift
@pytest.mark.parametrize("name,n,moduli,t,word_bits", U64, ids=ids(U64))
def test_plaintext_to_eval_at_lift_threshold(name, n, moduli, t, word_bits):
    g, o, _ = contexts(n, moduli, t, word_bits)
    plain = lift_plaintexts(n, t, t + 4)
    for l in range(o.L, 0, -1):
        want = np.stack([o.plaintext_to_eval(p, l) for p in plain])
        assert np.array_equal(hecuda.Bfv.plaintextToEval(g, plain, l), want), l
    g.close()


@pytest.mark.parametrize("name,n,moduli,t,word_bits", SIMD, ids=ids(SIMD))
def test_encode_simd_at_lift_threshold(name, n, moduli, t, word_bits):
    """encodeSimd of the slot values whose Coeff plaintexts hold the lift inputs, in Coeff and at every level in Eval."""
    g, o, bfv = contexts(n, moduli, t, word_bits)
    plain = lift_plaintexts(n, t, t + 5)
    slots = np.stack([pt.simd_values_for_coeff(o, p) for p in plain])
    assert np.array_equal(bfv.encodeSimd(g, words(slots, word_bits)).astype(np.uint64), plain)
    for l in range(o.L, 0, -1):
        want = np.stack([o.plaintext_to_eval(p, l) for p in plain])
        assert np.array_equal(bfv.encodeSimd(g, words(slots, word_bits), moduliCount=l).astype(np.uint64), want), l
    g.close()


@pytest.mark.parametrize("name,n,moduli,t,word_bits", pt.CONTEXTS, ids=pt.IDS)
def test_mulpir_database_at_lift_threshold(name, n, moduli, t, word_bits):
    """One plaintext per entry, whose bytes pack the lift inputs below 2^floor(log2 t) into its coefficients: the
    resident Eval rows of the host and the device processing both equal the oracle's lift of those plaintexts."""
    g, o, _ = contexts(n, moduli, t, word_bits)
    bits = t.bit_length() - 1
    values = [v for v in pt.lift_inputs(t) if v < 1 << bits]
    thr = pt.threshold(t)
    assert {thr - 1, thr} <= set(values) and (thr + 1 in values or thr + 1 >= 1 << bits)
    plain, _ = pt.threshold_polys(values, n, 1 << bits, random.Random(t + 6))
    db = [pir.CoefficientPacking.coefficientsToBytes(p.tolist(), bits) for p in plain]
    size = pir.bytesPerPlaintext(g)
    assert all(len(entry) == size for entry in db)
    param = pir.MulPir.generateParameter(pir.IndexPirConfig(len(db), size, 1, 1, False, "noCompression", False), g)
    rows, present = pir.MulPirServer.plaintextRows(db, g, param)
    assert np.array_equal(rows[:len(db)], plain) and not rows[len(db):].any()
    want = np.stack([o.plaintext_to_eval(r, o.L) for r in rows])
    host, device = pir.MulPirServer.process(db, g, param), pir.MulPirServer.processOnDevice(db, g, param)
    for db_ in (host, device):
        ptr, nbytes = db_.deviceBuffer()
        resident = read_device(ptr, nbytes)
        if nbytes == want.size * 4:  # uint32 rows when every ciphertext modulus is below 2^31
            resident = resident.view(np.uint32)
        assert np.array_equal(resident.astype(np.uint64).reshape(want.shape), want), db_ is device
        assert np.array_equal(db_.presentFlags(), present)
    host.close(), device.close()
    g.close()


# -------------------------------------------------------------------------------------------------------- D3 uncentre
@pytest.mark.parametrize("name,n,moduli,t,word_bits", SIMD, ids=ids(SIMD))
def test_decode_eval_at_uncentring_threshold(name, n, moduli, t, word_bits):
    """decodeSimd(moduliCount: l) of the Eval forms (valid lifts) of plaintexts holding thr - 1, thr and thr + 1 at
    every level: the slot values round-trip and equal the oracle's decode."""
    g, o, bfv = contexts(n, moduli, t, word_bits)
    plain = lift_plaintexts(n, t, t + 7)
    slots = np.stack([pt.simd_values_for_coeff(o, p) for p in plain])
    for l in range(o.L, 0, -1):
        ev = np.stack([o.plaintext_to_eval(p, l) for p in plain])
        want = np.stack([pn.decode_simd(o, ref.plaintext_to_coeff(n, moduli[0], t, e)) for e in ev])
        assert np.array_equal(want, slots), l
        got = bfv.decodeSimd(g, words(ev, word_bits), moduliCount=l).astype(np.uint64)
        assert np.array_equal(got, want), l
    g.close()
