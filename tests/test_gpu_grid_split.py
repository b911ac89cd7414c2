"""Device-pointer calls that hand one launcher more than 65535 items, which it puts in grid y or z (at most 65535):
the launcher runs the batch in parts.  N = 1024, one call of 70000 items per entry point, checked bit-exactly against
the oracle on both sides of the part boundary, with the call's kernel-launch count.

These are the `_device` calls that pass their whole batch to such a launcher; encode / decode / plaintext translate
are in test_gpu_plaintext.py.  The batched calls that chunk by the context's chunk size (at most 4096 ciphertexts)
never reach the limit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda
from oracle import oracle as orc
from oracle import pir_oracle as opir

N, T = 1024, 12289
COUNT = 70000  # two parts: 65535 and 4465
PROBES = (0, 65534, 65535, 65536, COUNT - 1)
BASE_Q = 0  # HECUDA_BASE_Q


@pytest.fixture(scope="module")
def ctx():
    moduli = orc.generate_primes([55, 55], False, N)
    g, o = hecuda.Context(N, moduli, T), orc.Context(N, moduli, T)
    assert o.L == 1
    yield g, o, moduli[:1]
    g.close()


def _uniform(bound, shape, seed):
    import torch

    gen = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, int(bound), shape, dtype=torch.int64, device="cuda", generator=gen)


def _launches(call):
    """kernel launches of one C-ABI call (it must succeed)"""
    before = hecuda.kernel_launch_count()
    hecuda._check(call())
    return hecuda.kernel_launch_count() - before


def _np(x):
    return x.cpu().numpy().view(np.uint64)


def _stream():
    import torch

    return torch.cuda.current_stream().cuda_stream


@pytest.mark.parametrize("op", ["add", "sub", "mul", "neg", "mul_scalars"])
def test_elementwise_past_grid_limit(ctx, op):
    g, o, q = ctx
    lib, s = hecuda.load_library(), _stream()
    scalars = np.array([int(q[0]) - 3], dtype=np.uint64)  # a host array, also for the _device variant
    fn = getattr(lib, f"hecuda_poly_{op}_device")

    def call(a, b, count):
        if op == "neg":
            return lambda: fn(g._h, BASE_Q, a.data_ptr(), 1, count, s)
        if op == "mul_scalars":
            return lambda: fn(g._h, BASE_Q, a.data_ptr(), scalars.ctypes.data, 1, count, s)
        return lambda: fn(g._h, BASE_Q, a.data_ptr(), b.data_ptr(), 1, count, s)

    a, b = _uniform(q[0], (COUNT, 1, N), 1), _uniform(q[0], (COUNT, 1, N), 2)
    before = _np(a)
    single = _launches(call(a[:1].clone(), b[:1].clone(), 1))
    # one split stage: the elementwise kernel (polynomials in grid z)
    assert _launches(call(a, b, COUNT)) == single + 1
    got, rhs, m = _np(a), _np(b), int(q[0])
    for i in PROBES:
        if op in ("add", "sub", "mul"):
            want = orc.poly_op(op, N, q, before[i], rhs[i])
        elif op == "neg":
            want = np.array([[(m - int(v)) % m for v in before[i, 0]]], dtype=np.uint64)
        else:
            want = np.array([[int(v) * int(scalars[0]) % m for v in before[i, 0]]], dtype=np.uint64)
        assert np.array_equal(got[i], want), (op, i)


def test_serialize_and_load_past_grid_limit(ctx):
    import torch

    g, o, q = ctx
    lib, s, skip = hecuda.load_library(), _stream(), 3
    size = hecuda.Bfv.serializationByteCount(g, 1, skip)
    x = _uniform(q[0], (COUNT, 1, N), 3)
    data = torch.empty((COUNT, size), dtype=torch.uint8, device="cuda")
    back = torch.empty_like(x)
    serialize = lambda d, out, count: lambda: lib.hecuda_poly_serialize_device(g._h, BASE_Q, d.data_ptr(), skip,
                                                                             out.data_ptr(), 1, count, s)
    load = lambda d, out, count: lambda: lib.hecuda_poly_load_device(g._h, BASE_Q, d.data_ptr(), skip, out.data_ptr(), 1,
                                                                   count, s)
    single = (_launches(serialize(x[:1], torch.empty_like(data[:1]), 1)),
              _launches(load(data[:1].clone(), torch.empty_like(back[:1]), 1)))
    # one split stage each: the serialize kernel and the load kernel (polynomials in grid z)
    assert _launches(serialize(x, data, COUNT)) == single[0] + 1
    assert _launches(load(data, back, COUNT)) == single[1] + 1
    polys, wire, loaded = _np(x), data.cpu().numpy(), _np(back)
    for i in PROBES:
        assert wire[i].tobytes() == opir.serialize_poly(N, q, polys[i], skip), i
        assert np.array_equal(loaded[i], opir.load_poly(N, q, wire[i].tobytes(), skip)), i


def test_plaintext_to_eval_past_grid_limit(ctx):
    import torch

    g, o, q = ctx
    lib, s = hecuda.load_library(), _stream()
    plain = _uniform(T, (COUNT, N), 4)
    out = torch.empty((COUNT, 1, N), dtype=torch.int64, device="cuda")
    call = lambda p, dst, count: lambda: lib.hecuda_plaintext_to_eval_device(g._h, p.data_ptr(), 1, dst.data_ptr(), count, s)
    single = _launches(call(plain[:1], torch.empty_like(out[:1]), 1))
    # one split stage: the centred lift (plaintexts in grid z); the forward NTT that follows is one launch at any count
    assert _launches(call(plain, out, COUNT)) == single + 1
    p, got = _np(plain), _np(out)
    for i in PROBES:
        assert np.array_equal(got[i], o.plaintext_to_eval(p[i], 1)), i


def test_inner_product_plaintexts_past_grid_limit(ctx):
    import torch

    g, o, q = ctx
    lib, s, terms = hecuda.load_library(), _stream(), 2
    cts = _uniform(q[0], (terms, 2, 1, N), 5)
    pts = _uniform(q[0], (COUNT, terms, 1, N), 6)
    out = torch.empty((COUNT, 2, 1, N), dtype=torch.int64, device="cuda")
    call = lambda p, dst, count: lambda: lib.hecuda_bfv_inner_product_plaintexts_device(
        g._h, cts.data_ptr(), 2, 1, terms, p.data_ptr(), None, dst.data_ptr(), count, s)
    single = _launches(call(pts[:1], torch.empty_like(out[:1]), 1))
    # one split stage: the scan (output rows in grid z)
    assert _launches(call(pts, out, COUNT)) == single + 1
    c, p, got = _np(cts), _np(pts), _np(out)
    for i in PROBES:
        assert np.array_equal(got[i], o.inner_product_plain(c, p[i:i + 1])[0]), i
