"""GPU parity of the plaintext side of Bfv -- SIMD encode / decode and ciphertext +- plaintext -- bit-exact against the
oracle (pnns_oracle.encode_simd / decode_simd, Context.plaintext_to_eval) and the restatements in tests/plaintext_ref.py,
at the reference's predefined parameter sets with an NTT-friendly t (EncryptionParameters.swift:272-449) plus N = 1024,
16384 and 32768 and Bfv<UInt32> contexts."""
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda
from oracle import oracle as orc
from oracle import pnns_oracle as pn
import plaintext_ref as ref

Q4096 = [134176769, 268369921, 268361729]                                      # 27/28/28 bits
Q8192_55 = [36028797018652673, 36028797017571329, 36028797017456641]          # 3 x 55 bits
PREDEFINED = [
    (4096, Q4096, 40961),
    (4096, Q4096, 65537),
    (8192, [268369921, 1152921504606830593, 1152921504606748673], 557057),
    (8192, Q8192_55, 8404993),
    (8192, Q8192_55, 268582913),
    (8192, Q8192_55, 536903681),
    (8192, Q8192_55, 2199023288321),
    (8192, [1099511480321, 1152921504606830593, 1152921504606748673], 33832961),
]
EXTRA = [(1024, [55, 55, 55], 12289), (16384, [55, 55, 55, 55], 786433), (32768, [55, 55, 55], 786433)]
CONTEXTS = PREDEFINED + [(n, orc.generate_primes(bits, False, n), t) for n, bits, t in EXTRA]
IDS = [f"n{n}-t{t}" for n, _, t in CONTEXTS]
WORD32 = [(4096, Q4096, 40961), (4096, Q4096, 65537)]  # Bfv<UInt32>: every modulus and t below 2^30
OPS = {ref.ADD: "addAssignCoeff", ref.SUB: "subAssignCoeff", ref.SUB_FROM: "subCoeff"}


def _contexts(n, moduli, t, word32=False):
    g = hecuda.Context(n, moduli, t, scalar=np.uint32 if word32 else np.uint64)
    return g, orc.Context(n, moduli, t, word_bits=32 if word32 else 64)


def _values(rng, t, shape):
    return np.array([rng.randrange(t) for _ in range(int(np.prod(shape)))], dtype=np.uint64).reshape(shape)


def _translate(bfv, g, op, ct, pt, out=None):
    if op == ref.SUB_FROM:
        return bfv.subCoeff(g, pt, ct, out=out)
    return getattr(bfv, OPS[op])(g, ct, pt, out=out)


@pytest.mark.parametrize("n,moduli,t", CONTEXTS, ids=IDS)
def test_encode_decode_match_oracle(n, moduli, t):
    g, o = _contexts(n, moduli, t)
    assert g.supportsSimdEncoding
    rng = random.Random(t)
    for count in (n // 2, n):
        values = _values(rng, t, (2, count))
        coeff = hecuda.Bfv.encodeSimd(g, values)
        want = np.stack([pn.encode_simd(o, v) for v in values])
        assert np.array_equal(coeff, want), count
        padded = np.concatenate([values, np.zeros((2, n - count), dtype=np.uint64)], axis=1)
        assert np.array_equal(hecuda.Bfv.decodeSimd(g, coeff), padded)
        for l in range(1, o.L + 1):
            ev = hecuda.Bfv.encodeSimd(g, values, moduliCount=l)
            assert np.array_equal(ev, np.stack([o.plaintext_to_eval(p, l) for p in want])), (count, l)
            assert np.array_equal(hecuda.Bfv.decodeSimd(g, ev, moduliCount=l), padded), (count, l)
    # one unbatched value vector: (valueCount,) -> (N,)
    assert np.array_equal(hecuda.Bfv.encodeSimd(g, values[0]), want[0])
    g.close()


@pytest.mark.parametrize("n,moduli,t", CONTEXTS, ids=IDS)
def test_translate_matches_reference(n, moduli, t):
    g, o = _contexts(n, moduli, t)
    rng = random.Random(n ^ t)
    batch = 3
    for l in range(o.L, 0, -1):
        for polys in (2, 3):
            ct = orc.fill_uniform(polys * l + l, moduli[:l], n, batch * polys * l).reshape(batch, polys, l, n)
            pts = _values(rng, t, (batch, n))
            for op in OPS:
                per = np.stack([ref.plaintext_translate(moduli, t, ct[i], pts[i], op) for i in range(batch)])
                shared = np.stack([ref.plaintext_translate(moduli, t, ct[i], pts[0], op) for i in range(batch)])
                assert np.array_equal(_translate(hecuda.Bfv, g, op, ct, pts), per), (l, polys, op)
                assert np.array_equal(_translate(hecuda.Bfv, g, op, ct, pts[0]), shared), (l, polys, op)
                inplace = ct.copy()
                assert _translate(hecuda.Bfv, g, op, inplace, pts, out=inplace) is inplace
                assert np.array_equal(inplace, per), (l, polys, op, "in place")
    g.close()


@pytest.mark.parametrize("t", [65537, 2199023288321])
def test_translate_device_in_place_and_out_of_place(t):
    import torch

    n, moduli = (4096, Q4096) if t < 2 ** 30 else (8192, Q8192_55)
    g, o = _contexts(n, moduli, t)
    rng = random.Random(t)
    l, polys, batch = o.L, 3, 4
    ct = orc.fill_uniform(9, moduli[:l], n, batch * polys * l).reshape(batch, polys, l, n)
    pts = _values(rng, t, (batch, n))
    lib, s = hecuda.load_library(), torch.cuda.current_stream().cuda_stream
    for op in OPS:
        want = np.stack([ref.plaintext_translate(moduli, t, ct[i], pts[i], op) for i in range(batch)])
        d_ct, d_pt = torch.from_numpy(ct.view(np.int64)).cuda(), torch.from_numpy(pts.view(np.int64)).cuda()
        d_out = torch.empty_like(d_ct)
        hecuda._check(lib.hecuda_bfv_plaintext_translate_device(g._h, d_ct.data_ptr(), polys, l, d_pt.data_ptr(), batch, op,
                                                                d_out.data_ptr(), batch, s))
        hecuda._check(lib.hecuda_bfv_plaintext_translate_device(g._h, d_ct.data_ptr(), polys, l, d_pt.data_ptr(), batch, op,
                                                                d_ct.data_ptr(), batch, s))
        torch.cuda.synchronize()
        assert np.array_equal(d_out.cpu().numpy().view(np.uint64), want), op
        assert np.array_equal(d_ct.cpu().numpy().view(np.uint64), want), (op, "in place")
    g.close()


@pytest.mark.parametrize("n,moduli,t", WORD32, ids=[f"u32-t{t}" for _, _, t in WORD32])
def test_word32_matches_word64(n, moduli, t):
    g, o = _contexts(n, moduli, t, word32=True)
    rng = random.Random(t + 1)
    values = _values(rng, t, (3, n))
    want = np.stack([pn.encode_simd(o, v) for v in values])
    coeff = hecuda.Bfv32.encodeSimd(g, values)
    assert coeff.dtype == np.uint32 and np.array_equal(coeff.astype(np.uint64), want)
    assert np.array_equal(hecuda.Bfv32.decodeSimd(g, coeff).astype(np.uint64), values)
    for l in range(1, o.L + 1):
        ev = hecuda.Bfv32.encodeSimd(g, values, moduliCount=l)
        assert np.array_equal(ev.astype(np.uint64), np.stack([o.plaintext_to_eval(p, l) for p in want]))
        assert np.array_equal(hecuda.Bfv32.decodeSimd(g, ev, moduliCount=l).astype(np.uint64), values)
        for polys in (2, 3):
            ct = orc.fill_uniform(l + polys, moduli[:l], n, 3 * polys * l).reshape(3, polys, l, n)
            for op in OPS:
                want_ct = np.stack([ref.plaintext_translate(moduli, t, ct[i], want[i], op) for i in range(3)])
                got = _translate(hecuda.Bfv32, g, op, ct.astype(np.uint32), want.astype(np.uint32))
                assert got.dtype == np.uint32 and np.array_equal(got.astype(np.uint64), want_ct), (l, polys, op)
                got = _translate(hecuda.Bfv32, g, op, ct.astype(np.uint32), want[0].astype(np.uint32))
                assert np.array_equal(got[1].astype(np.uint64), ref.plaintext_translate(moduli, t, ct[1], want[0], op))
    g.close()


@pytest.mark.parametrize("n,moduli,t", [(8192, [268369921, 1152921504606830593, 1152921504606748673], 557057),
                                        (8192, Q8192_55, 2199023288321)], ids=["t557057", "t2199023288321"])
def test_end_to_end_encrypt_translate_decrypt_decode(n, moduli, t):
    """oracle-encrypt encode(a) -> GPU translate with encode(b) -> GPU decrypt -> GPU decode = a +- b mod t."""
    g, o = _contexts(n, moduli, t)
    rng = random.Random(5)
    sk, _ = o.keygen(6, relin=False)
    a, b = _values(rng, t, (n,)), _values(rng, t, (n,))
    ct = o.encrypt(21, sk, hecuda.Bfv.encodeSimd(g, a))[None]
    pb = hecuda.Bfv.encodeSimd(g, b)
    ao, bo = a.astype(object), b.astype(object)
    for l in range(o.L, 0, -1):
        for op, want in ((ref.ADD, (ao + bo) % t), (ref.SUB, (ao - bo) % t), (ref.SUB_FROM, (bo - ao) % t)):
            dec = hecuda.Bfv.decrypt(g, _translate(hecuda.Bfv, g, op, ct, pb), sk)
            assert np.array_equal(hecuda.Bfv.decodeSimd(g, dec)[0].astype(object), want), (l, op)
        if l > 1:
            ct = o.mod_switch_down(ct)
    g.close()


def test_errors():
    n = 4096
    g, o = _contexts(n, Q4096, 17)  # t = 17 is not 1 mod 2N: no SIMD encoding
    assert not g.supportsSimdEncoding
    with pytest.raises(hecuda.HeError) as e:
        hecuda.Bfv.encodeSimd(g, [1, 2, 3])
    assert e.value.code == -2 and "simdEncodingNotSupported" in e.value.message
    with pytest.raises(hecuda.HeError) as e:
        hecuda.Bfv.decodeSimd(g, np.zeros(n, dtype=np.uint64))
    assert e.value.code == -2
    # ... while ciphertext +- plaintext still works
    ct = orc.fill_uniform(1, Q4096[:2], n, 4).reshape(1, 2, 2, n)
    m = np.arange(n, dtype=np.uint64) % 17
    assert np.array_equal(hecuda.Bfv.addAssignCoeff(g, ct, m)[0], ref.plaintext_translate(Q4096, 17, ct[0], m, ref.ADD))
    with pytest.raises(hecuda.HeError):
        hecuda.Bfv.addAssignCoeff(g, ct, m + 17)  # coefficient >= t
    g.close()

    g = hecuda.Context(n, Q4096, 65537)
    with pytest.raises(hecuda.HeError) as e:
        hecuda.Bfv.encodeSimd(g, np.zeros(n + 1, dtype=np.uint64))
    assert e.value.code == -1 and "encodingDataCountExceedsLimit" in e.value.message
    with pytest.raises(hecuda.HeError) as e:
        hecuda.Bfv.encodeSimd(g, [0, 65537])
    assert e.value.code == -1 and "encodingDataOutOfBounds" in e.value.message
    with pytest.raises(hecuda.HeError):
        hecuda.Bfv.encodeSimd(g, [1], moduliCount=g.L + 1)
    ct = np.zeros((1, 2, 2, n), dtype=np.uint64)
    lib = hecuda.load_library()
    pt = np.zeros(n, dtype=np.uint64)
    for polys, l, count, op in ((4, 2, 1, 0), (2, 0, 1, 0), (2, 3, 1, 0), (2, 2, 2, 0), (2, 2, 1, 3)):
        rc = lib.hecuda_bfv_plaintext_translate(g._h, hecuda._ptr(ct), polys, l, hecuda._ptr(pt), count, op, hecuda._ptr(ct), 1)
        assert rc == -1, (polys, l, count, op)
    g.close()


def test_batch_above_grid_limit_n1024():
    """One device-pointer call with more than 65535 plaintexts / ciphertexts at N = 1024."""
    import torch

    n, t = 1024, 12289
    moduli = orc.generate_primes([55, 55], False, n)
    g, o = _contexts(n, moduli, t)
    count = 70000
    values = torch.randint(0, t, (count, n), dtype=torch.int64, device="cuda")
    lib, s = hecuda.load_library(), torch.cuda.current_stream().cuda_stream
    coeff = torch.empty_like(values)
    ev = torch.empty_like(values)
    back = torch.empty_like(values)
    hecuda._check(lib.hecuda_bfv_encode_simd_device(g._h, values.data_ptr(), n, 0, coeff.data_ptr(), count, s))
    hecuda._check(lib.hecuda_bfv_encode_simd_device(g._h, values.data_ptr(), n, 1, ev.data_ptr(), count, s))
    hecuda._check(lib.hecuda_bfv_decode_simd_device(g._h, ev.data_ptr(), 1, back.data_ptr(), count, s))
    ct = torch.zeros((count, 2, 1, n), dtype=torch.int64, device="cuda")
    hecuda._check(lib.hecuda_bfv_plaintext_translate_device(g._h, ct.data_ptr(), 2, 1, coeff.data_ptr(), count,
                                                            ref.ADD, ct.data_ptr(), count, s))
    torch.cuda.synchronize()
    assert torch.equal(back, values)
    v, c, e, out = (x.cpu().numpy().view(np.uint64) for x in (values, coeff, ev, ct))
    for i in (0, 65534, 65535, 65536, count - 1):
        assert np.array_equal(c[i], pn.encode_simd(o, v[i])), i
        assert np.array_equal(e[i], o.plaintext_to_eval(c[i], 1)[0]), i
        assert np.array_equal(out[i], ref.plaintext_translate(moduli, t, np.zeros((2, 1, n), dtype=np.uint64), c[i], ref.ADD)), i
    g.close()


def test_plaintext_modulus_ntt_rows():
    """The context holds t's NTT tables (Context.plaintextContext): the row NTT entry points accept t."""
    n, t = 4096, 65537
    g, o = _contexts(n, Q4096, t)
    rows = _values(random.Random(1), t, (2, n))
    assert np.array_equal(hecuda.Bfv.forwardNttRows(g, t, rows), orc.ntt_forward(n, [t], rows))
    roots, _ = g.rootTables(t)
    assert np.array_equal(roots, orc.ntt_tables(n, t)[0])
    g.close()
