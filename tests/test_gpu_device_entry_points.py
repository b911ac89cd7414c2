"""The `_device` entry points of include/hecuda.h, called through the C ABI on torch device tensors the way bench.py calls
them.  Bit-exact throughout.

A. The benchmark's own workloads (bench.WORKLOADS): N, moduli, t and batch, inputs drawn like Harness.uniform, against
   the oracle.  The device calls loop over `h->chunk` items per launch sequence (hecuda_context_create sizes a chunk at
   about 2 GiB of multiply scratch); every batch here spans at least two such chunks, so chunk boundaries and the
   buffer offsets past them are exercised at the sizes the benchmark runs.
B. Stream semantics: each call is enqueued on a fresh stream that is still asleep and whose inputs arrive only after the
   sleep.  A call that synchronises, or that runs any kernel or copy on another stream, fails here every time.
C. Graph capture of the device calls, replayed with new inputs.
D. The N = 2^15 NTT past 65535 polynomials (grid z of the split / merge kernels).
E. The argument contract of the device calls: empty batches, NULL buffers, foreign and missing keys.

Tests that need more than 8 GiB of device memory check torch.cuda.mem_get_info() first and skip, stating what they
need, when the device does not have it free."""
import contextlib
import os
import threading

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import bench  # noqa: E402
import hecuda  # noqa: E402
from hecuda import pnns  # noqa: E402
from oracle import oracle as orc  # noqa: E402

GiB = 1 << 30
OK, ERR_INVALID_ARGUMENT, ERR_MISSING_KEY = 0, -1, -5
# ~200 ms of torch.cuda._sleep at the H100's 1.98 GHz boost clock (longer at lower clocks)
SLEEP_CYCLES = 400_000_000


def lib():
    return hecuda.load_library()


def ok(rc):
    hecuda._check(rc)


def device_chunk(n, L):
    """h->chunk as hecuda_context_create sizes it: 2 GiB of multiply scratch (7 (2L+1) N words per pair), at most 4096."""
    return max(1, min((2 << 30) // (7 * (2 * L + 1) * n * 8), 4096))


def require_free(nbytes, what):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"{what} needs {nbytes / GiB:.1f} GiB of free device memory; {free / GiB:.1f} GiB are free")


@contextlib.contextmanager
def chunk_env(chunk):
    """HECUDA_CHUNK as hecuda_context_create reads it (None: the default sizing rule)."""
    old = os.environ.pop("HECUDA_CHUNK", None)
    if chunk is not None:
        os.environ["HECUDA_CHUNK"] = str(chunk)
    try:
        yield
    finally:
        os.environ.pop("HECUDA_CHUNK", None)
        if old is not None:
            os.environ["HECUDA_CHUNK"] = old


def make_context(n, moduli, t, chunk=None, scalar=np.uint64):
    with chunk_env(chunk):
        return hecuda.Context(n, moduli, t, scalar=scalar)


def generator(seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return g


def uniform(gen, shape, moduli):
    """Harness.uniform: residues in [0, q_i) along the second-to-last axis."""
    qs = torch.tensor([int(q) for q in moduli], dtype=torch.int64, device="cuda").view(*([1] * (len(shape) - 2)), len(moduli), 1)
    x = torch.randint(0, 1 << 62, shape, generator=gen, device="cuda", dtype=torch.int64)
    return (x % qs).contiguous()


def host(t):
    return t.cpu().numpy().view(np.uint64)


def stream_ptr():
    return torch.cuda.current_stream().cuda_stream


def chunk_sample(batch, chunk, seed, extra=32):
    """The first and last 3 items of every device chunk, plus `extra` seeded indices."""
    idx = set()
    for start in range(0, batch, chunk):
        end = min(start + chunk, batch)
        idx.update(range(start, min(start + 3, end)))
        idx.update(range(max(start, end - 3), end))
    idx.update(int(i) for i in np.random.default_rng(seed).choice(batch, size=min(extra, batch), replace=False))
    return np.array(sorted(idx))


# ================================================================================ A. the benchmark's shapes vs the oracle
@pytest.mark.parametrize("name", ["C1", "C1-8192"])
def test_benchmark_ntt_matches_oracle_and_round_trips(name):
    n, moduli, t, batch = bench.workload_params(name)
    g = make_context(n, moduli, t)
    data = uniform(generator(101), (batch, 1, n), moduli[:1])
    x = data.clone()
    want = orc.ntt_forward_inplace(n, moduli[:1], host(data).copy(), orc.num_threads())
    ok(lib().hecuda_ntt_forward_device(g._h, hecuda.BASE_Q, data.data_ptr(), 1, batch, stream_ptr()))
    assert np.array_equal(host(data), want)
    ok(lib().hecuda_ntt_inverse_device(g._h, hecuda.BASE_Q, data.data_ptr(), 1, batch, stream_ptr()))
    assert torch.equal(data, x)
    g.close()


@pytest.mark.parametrize("name", ["C2", "C3"])
def test_roofline_ntt_shapes_match_oracle(name):
    """The launch shapes bench.ntt_roofline times: [Q, aux] with 2L+1 rows and min(batch, chunk) x 4 polynomials at C2,
    [Q, q_ks] with L+1 rows and 256 polynomials at C3; canonical residues of every row's own modulus."""
    n, moduli, t, batch = bench.workload_params(name)
    g = make_context(n, moduli, t)
    L = g.L
    if name == "C2":
        base, row_moduli, polys = hecuda.BASE_Q_AUX, moduli[:L] + g.auxModuli, min(batch, device_chunk(n, L)) * 4
    else:
        base, row_moduli, polys = hecuda.BASE_KEYSWITCH, moduli[:L] + [moduli[L]], min(batch, 256)
    rows = len(row_moduli)
    data = uniform(generator(102), (polys, rows, n), row_moduli)
    x = data.clone()
    want = orc.ntt_forward_inplace(n, row_moduli, host(data).copy(), orc.num_threads())
    ok(lib().hecuda_ntt_forward_device(g._h, base, data.data_ptr(), rows, polys, stream_ptr()))
    assert np.array_equal(host(data), want)
    ok(lib().hecuda_ntt_inverse_device(g._h, base, data.data_ptr(), rows, polys, stream_ptr()))
    assert torch.equal(data, x)
    g.close()


@pytest.mark.parametrize("name", ["C2", "C2-L4", "C2-u32"])
def test_benchmark_multiply_matches_oracle(name):
    """The whole batch of bench.run_mul's timed step; C2-u32 on a Bfv<UInt32> context in 64-bit slots, as benched."""
    n, moduli, t, batch = bench.workload_params(name)
    word32 = bench.WORKLOADS[name][0] == "mul32"
    g = make_context(n, moduli, t, scalar=np.uint32 if word32 else np.uint64)
    L = g.L
    assert batch > device_chunk(n, L), "the batch no longer spans two device chunks"
    gen = generator(103)
    lhs, rhs = uniform(gen, (batch, 2, L, n), moduli[:L]), uniform(gen, (batch, 2, L, n), moduli[:L])
    out = torch.empty((batch, 3, L, n), dtype=torch.int64, device="cuda")
    ok(lib().hecuda_bfv_multiply_device(g._h, lhs.data_ptr(), rhs.data_ptr(), out.data_ptr(), batch, stream_ptr()))
    o = orc.Context(n, moduli, t, word_bits=32 if word32 else 64)
    want = o.mul(host(lhs), host(rhs))
    got = host(out)
    bad = [i for i in range(batch) if not np.array_equal(got[i], want[i])]
    assert not bad, f"{len(bad)} of {batch} products differ, first {bad[:8]}"
    g.close()


def test_benchmark_c2_relinearize_and_fused_match_oracle():
    """bench.run_mul's extras: relinearize the product with a uniform synthetic key, and multiply + relinearize
    (+ modSwitchDown) in one call; the first and last items of every device chunk plus 32 seeded ones."""
    n, moduli, t, batch = bench.workload_params("C2")
    g = make_context(n, moduli, t)
    L, K = g.L, g.L + 1
    chunk = device_chunk(n, L)
    assert batch > chunk, "the batch no longer spans two device chunks"
    gen = generator(104)
    lhs, rhs = uniform(gen, (batch, 2, L, n), moduli[:L]), uniform(gen, (batch, 2, L, n), moduli[:L])
    key = host(uniform(gen, (L, 2, K, n), moduli))
    evk = hecuda.EvaluationKey(g, key)
    s = stream_ptr()
    prod = torch.empty((batch, 3, L, n), dtype=torch.int64, device="cuda")
    relin = torch.empty((batch, 2, L, n), dtype=torch.int64, device="cuda")
    fused = [torch.empty((batch, 2, L - m, n), dtype=torch.int64, device="cuda") for m in (0, 1)]
    ok(lib().hecuda_bfv_multiply_device(g._h, lhs.data_ptr(), rhs.data_ptr(), prod.data_ptr(), batch, s))
    ok(lib().hecuda_bfv_relinearize_device(g._h, evk._h, prod.data_ptr(), L, relin.data_ptr(), batch, s))
    for m in (0, 1):
        ok(lib().hecuda_bfv_multiply_relinearize_device(g._h, evk._h, lhs.data_ptr(), rhs.data_ptr(), m, fused[m].data_ptr(),
                                                        batch, s))
    idx = np.union1d(chunk_sample(batch, chunk, 1), chunk_sample(batch, chunk // 2, 2))
    sel = torch.from_numpy(idx).cuda()
    o = orc.Context(n, moduli, t)
    want_prod = o.mul(host(lhs.index_select(0, sel)), host(rhs.index_select(0, sel)))
    want_relin = o.relinearize(want_prod, key)
    assert np.array_equal(host(prod.index_select(0, sel)), want_prod)
    assert np.array_equal(host(relin.index_select(0, sel)), want_relin)
    assert np.array_equal(host(fused[0].index_select(0, sel)), want_relin)
    assert np.array_equal(host(fused[1].index_select(0, sel)), o.mod_switch_down(want_relin))
    evk.close()
    g.close()


def test_benchmark_c3_step_matches_oracle():
    """bench.run_relin's timed step over all 4096 ciphertexts: relinearize, then modSwitchDown of its output."""
    n, moduli, t, batch = bench.workload_params("C3")
    L, K = len(moduli) - 1, len(moduli)
    chunk = device_chunk(n, L)
    assert batch > chunk, "the batch no longer spans two device chunks"
    words = batch * (3 * L + 2 * L + 2 * (L - 1)) * n
    scratch = chunk * ((L + 1) * L + 2 * (L + 1)) * n
    require_free((words + scratch) * 8 + 2 * GiB, "the C3 step over 4096 ciphertexts")
    g = make_context(n, moduli, t)
    assert g.L == L
    gen = generator(105)
    ct3 = torch.empty((batch, 3, L, n), dtype=torch.int64, device="cuda")
    for start in range(0, batch, 512):  # in slices: uniform() holds two copies of what it draws
        ct3[start:start + 512] = uniform(gen, (min(512, batch - start), 3, L, n), moduli[:L])
    key = host(uniform(gen, (L, 2, K, n), moduli))
    evk = hecuda.EvaluationKey(g, key)
    relin = torch.empty((batch, 2, L, n), dtype=torch.int64, device="cuda")
    down = torch.empty((batch, 2, L - 1, n), dtype=torch.int64, device="cuda")
    s = stream_ptr()
    ok(lib().hecuda_bfv_relinearize_device(g._h, evk._h, ct3.data_ptr(), L, relin.data_ptr(), batch, s))
    ok(lib().hecuda_bfv_mod_switch_down_device(g._h, relin.data_ptr(), 2, L, down.data_ptr(), batch, s))
    sel = torch.from_numpy(chunk_sample(batch, chunk, 3)).cuda()
    o = orc.Context(n, moduli, t)
    want_relin = o.relinearize(host(ct3.index_select(0, sel)), key)
    assert np.array_equal(host(relin.index_select(0, sel)), want_relin)
    assert np.array_equal(host(down.index_select(0, sel)), o.mod_switch_down(want_relin))
    del ct3, relin, down
    evk.close()
    g.close()


def test_ragged_tails_match_oracle():
    """HECUDA_CHUNK=7 and a batch of 23: three full chunks and a tail of 2 (multiply_relinearize: chunks of 3 and 2)."""
    n, moduli, t, _ = bench.workload_params("C2")
    g = make_context(n, moduli, t, chunk=7)
    L, K, batch = g.L, g.L + 1, 23
    gen = generator(106)
    lhs, rhs = uniform(gen, (batch, 2, L, n), moduli[:L]), uniform(gen, (batch, 2, L, n), moduli[:L])
    key = host(uniform(gen, (L, 2, K, n), moduli))
    evk = hecuda.EvaluationKey(g, key)
    s = stream_ptr()
    prod = torch.empty((batch, 3, L, n), dtype=torch.int64, device="cuda")
    relin = torch.empty((batch, 2, L, n), dtype=torch.int64, device="cuda")
    fused = [torch.empty((batch, 2, L - m, n), dtype=torch.int64, device="cuda") for m in (0, 1)]
    ok(lib().hecuda_bfv_multiply_device(g._h, lhs.data_ptr(), rhs.data_ptr(), prod.data_ptr(), batch, s))
    ok(lib().hecuda_bfv_relinearize_device(g._h, evk._h, prod.data_ptr(), L, relin.data_ptr(), batch, s))
    for m in (0, 1):
        ok(lib().hecuda_bfv_multiply_relinearize_device(g._h, evk._h, lhs.data_ptr(), rhs.data_ptr(), m, fused[m].data_ptr(),
                                                        batch, s))
    o = orc.Context(n, moduli, t)
    want_prod = o.mul(host(lhs), host(rhs))
    want_relin = o.relinearize(want_prod, key)
    assert np.array_equal(host(prod), want_prod)
    assert np.array_equal(host(relin), want_relin)
    assert np.array_equal(host(fused[0]), want_relin)
    assert np.array_equal(host(fused[1]), o.mod_switch_down(want_relin))
    evk.close()
    g.close()


# ================================================================================ B. the caller's stream
_TORCH = {np.dtype(np.uint64): torch.int64, np.dtype(np.uint8): torch.uint8}


def _as_torch(a):
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a)


def _as_numpy(t, dtype):
    a = t.numpy()
    return a.view(np.uint64) if np.dtype(dtype) == np.uint64 else a


def run_on_busy_stream(inputs, outputs, call):
    """Warm up once, then: a fresh stream sleeps, the inputs are copied onto it (pinned host -> device, non-blocking),
    `call(device_inputs, device_outputs, stream)` enqueues, the stream must still be busy when the call returns, the
    results are copied out on that stream and only it is synchronised.  Returns the host copies of the inputs (after
    the call: some calls work in place) and of the outputs."""
    d_in = [torch.zeros(a.shape, dtype=_TORCH[a.dtype], device="cuda") for a in inputs]
    d_out = [torch.zeros(shape, dtype=_TORCH[np.dtype(dt)], device="cuda") for shape, dt in outputs]
    pinned = [_as_torch(a).pin_memory() for a in inputs]
    for d, p in zip(d_in, pinned):
        d.copy_(p)
    ok(call(d_in, d_out, stream_ptr()))  # first-call attribute setup and scratch pool growth happen here
    torch.cuda.synchronize()
    for d in d_in + d_out:
        d.zero_()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        for d, p in zip(d_in, pinned):
            d.copy_(p, non_blocking=True)
    ok(call(d_in, d_out, s.cuda_stream))
    busy = not s.query()
    results = [torch.empty(d.shape, dtype=d.dtype, pin_memory=True) for d in d_in + d_out]
    with torch.cuda.stream(s):
        for r, d in zip(results, d_in + d_out):
            r.copy_(d, non_blocking=True)
    s.synchronize()
    assert busy, "the call returned after its stream had drained: it synchronised"
    dtypes = [a.dtype for a in inputs] + [np.dtype(dt) for _, dt in outputs]
    got = [_as_numpy(r, dt) for r, dt in zip(results, dtypes)]
    return got[:len(inputs)], got[len(inputs):]


STREAM_N = 4096
STREAM_CHUNK = 2  # HECUDA_CHUNK: batches of 5 run as chunks of 2, 2 and 1 (multiply_relinearize: 1 item per chunk)
STREAM_BATCH = 5


@pytest.fixture(scope="module")
def small():
    n = STREAM_N
    moduli = orc.generate_primes([55] * 4, False, n)
    t = 65537  # prime = 1 mod 2N: SIMD encoding for the PNNS matrix
    g = make_context(n, moduli, t, chunk=STREAM_CHUNK)
    L, K = g.L, g.L + 1
    rng = np.random.default_rng(7)

    def residues(shape, mods):
        q = np.array(mods, dtype=np.uint64).reshape(len(mods), 1)
        return (rng.integers(0, 1 << 62, size=shape, dtype=np.uint64) % q).astype(np.uint64)

    relin_key = residues((L, 2, K, n), moduli)
    evk = hecuda.EvaluationKey(g, relin_key)
    element = pnns.GaloisElement.rotatingColumns(-1, n)
    elements = [element]
    cols = 16
    bsgs = pnns.BabyStepGiantStep.forVectorDimension(cols)
    if bsgs.giantStep > 1:
        elements.append(pnns.GaloisElement.rotatingColumns(-bsgs.babyStep, n))
    for e in dict.fromkeys(elements):
        evk.setGaloisKey(e, residues((L, 2, K, n), moduli))
    rows = 100
    matrix = pnns.PlaintextMatrix(g, pnns.MatrixDimensions(rows, cols), [int(v) for v in rng.integers(0, t, rows * cols)])
    yield dict(g=g, n=n, moduli=moduli, t=t, L=L, evk=evk, element=element, matrix=matrix, residues=residues, rng=rng)
    matrix.close()
    evk.close()
    g.close()


def _stream_case(name, S):
    """(inputs, outputs, call, expected outputs or in-place inputs) of one device entry point on the small context."""
    g, n, L, t, B = S["g"], S["n"], S["L"], S["t"], STREAM_BATCH
    q = S["moduli"][:L]
    res, rng, evk = S["residues"], S["rng"], S["evk"]
    Q = hecuda.BASE_Q
    U64 = np.uint64
    if name in ("ntt_forward", "ntt_inverse"):
        x = res((B, L, n), q)
        fn = getattr(lib(), f"hecuda_{name}_device")
        want = (hecuda.Bfv.forwardNtt if name == "ntt_forward" else hecuda.Bfv.inverseNtt)(g, x, Q)
        return [x], [], lambda i, o, s: fn(g._h, Q, i[0].data_ptr(), L, B, s), ("in", [want])
    if name == "multiply":
        a, b = res((B, 2, L, n), q), res((B, 2, L, n), q)
        return ([a, b], [((B, 3, L, n), U64)],
                lambda i, o, s: lib().hecuda_bfv_multiply_device(g._h, i[0].data_ptr(), i[1].data_ptr(), o[0].data_ptr(), B, s),
                ("out", [hecuda.Bfv.mulAssign(g, a, b)]))
    if name == "relinearize":
        c = res((B, 3, L, n), q)
        return ([c], [((B, 2, L, n), U64)],
                lambda i, o, s: lib().hecuda_bfv_relinearize_device(g._h, evk._h, i[0].data_ptr(), L, o[0].data_ptr(), B, s),
                ("out", [hecuda.Bfv.relinearize(g, c, evk)]))
    if name == "mod_switch_down":
        c = res((B, 2, L, n), q)
        return ([c], [((B, 2, L - 1, n), U64)],
                lambda i, o, s: lib().hecuda_bfv_mod_switch_down_device(g._h, i[0].data_ptr(), 2, L, o[0].data_ptr(), B, s),
                ("out", [hecuda.Bfv.modSwitchDown(g, c)]))
    if name.startswith("multiply_relinearize"):
        m = int(name[-1])
        a, b = res((B, 2, L, n), q), res((B, 2, L, n), q)
        return ([a, b], [((B, 2, L - m, n), U64)],
                lambda i, o, s: lib().hecuda_bfv_multiply_relinearize_device(g._h, evk._h, i[0].data_ptr(), i[1].data_ptr(), m,
                                                                             o[0].data_ptr(), B, s),
                ("out", [hecuda.Bfv.mulRelinearize(g, a, b, evk, modSwitchDown=bool(m))]))
    if name == "apply_galois":
        c, e = res((B, 2, L, n), q), S["element"]
        return ([c], [((B, 2, L, n), U64)],
                lambda i, o, s: lib().hecuda_bfv_apply_galois_device(g._h, evk._h, i[0].data_ptr(), L, e, o[0].data_ptr(), B, s),
                ("out", [hecuda.Bfv.applyGalois(g, c, e, evk)]))
    if name == "inner_product":
        pairs, groups = 3, 3  # chunks of max(1, 2 / 3) = 1 group
        a, b = res((groups, pairs, 2, L, n), q), res((groups, pairs, 2, L, n), q)
        return ([a, b], [((groups, 3, L, n), U64)],
                lambda i, o, s: lib().hecuda_bfv_inner_product_device(g._h, i[0].data_ptr(), i[1].data_ptr(), o[0].data_ptr(),
                                                                      pairs, groups, s),
                ("out", [hecuda.Bfv.innerProductCiphertexts(g, a, b)]))
    if name.startswith("inner_product_plaintexts"):
        terms, rows = 6, 4
        cts, pts = res((terms, 2, L, n), q), res((rows, terms, L, n), q)
        if name.endswith("mask"):
            present = (rng.integers(0, 3, size=(rows, terms)) > 0).astype(np.uint8)
            present[0, 0] = present[1, -1] = present[2, :] = 0
            return ([cts, pts, present], [((rows, 2, L, n), U64)],
                    lambda i, o, s: lib().hecuda_bfv_inner_product_plaintexts_device(
                        g._h, i[0].data_ptr(), 2, L, terms, i[1].data_ptr(), i[2].data_ptr(), o[0].data_ptr(), rows, s),
                    ("out", [hecuda.Bfv.innerProduct(g, cts, pts, present)]))
        return ([cts, pts], [((rows, 2, L, n), U64)],
                lambda i, o, s: lib().hecuda_bfv_inner_product_plaintexts_device(
                    g._h, i[0].data_ptr(), 2, L, terms, i[1].data_ptr(), None, o[0].data_ptr(), rows, s),
                ("out", [hecuda.Bfv.innerProduct(g, cts, pts)]))
    if name == "plaintext_to_eval":
        count = 6
        plain = rng.integers(0, t, size=(count, n), dtype=np.uint64)
        return ([plain], [((count, L, n), U64)],
                lambda i, o, s: lib().hecuda_plaintext_to_eval_device(g._h, i[0].data_ptr(), L, o[0].data_ptr(), count, s),
                ("out", [hecuda.Bfv.plaintextToEval(g, plain, L)]))
    if name in ("poly_add", "poly_sub", "poly_mul"):
        a, b = res((B, L, n), q), res((B, L, n), q)
        fn = getattr(lib(), f"hecuda_{name}_device")
        want = {"poly_add": hecuda.Bfv.polyAdd, "poly_sub": hecuda.Bfv.polySub, "poly_mul": hecuda.Bfv.polyMul}[name](g, a, b)
        return [a, b], [], lambda i, o, s: fn(g._h, Q, i[0].data_ptr(), i[1].data_ptr(), L, B, s), ("in", [want, b])
    if name == "poly_neg":
        a = res((B, L, n), q)
        return ([a], [], lambda i, o, s: lib().hecuda_poly_neg_device(g._h, Q, i[0].data_ptr(), L, B, s),
                ("in", [hecuda.Bfv.polyNeg(g, a)]))
    if name == "poly_mul_scalars":
        a = res((B, L, n), q)
        scalars = np.array([int(v) % p for v, p in zip(rng.integers(1, 1 << 62, size=L, dtype=np.uint64), q)], dtype=np.uint64)
        # scalars is a host array, also for the _device variant (include/hecuda.h)
        return ([a], [], lambda i, o, s: lib().hecuda_poly_mul_scalars_device(g._h, Q, i[0].data_ptr(), scalars.ctypes.data, L, B, s),
                ("in", [hecuda.Bfv.polyMulScalars(g, a, scalars)]))
    if name == "poly_serialize":
        a, skip = res((B, L, n), q), 3
        size = hecuda.Bfv.serializationByteCount(g, L, skip)
        return ([a], [((B, size), np.uint8)],
                lambda i, o, s: lib().hecuda_poly_serialize_device(g._h, Q, i[0].data_ptr(), skip, o[0].data_ptr(), L, B, s),
                ("out", [hecuda.Bfv.serialize(g, a, skip)]))
    if name == "poly_load":
        skip = 3
        data = hecuda.Bfv.serialize(g, res((B, L, n), q), skip)
        return ([data], [((B, L, n), U64)],
                lambda i, o, s: lib().hecuda_poly_load_device(g._h, Q, i[0].data_ptr(), skip, o[0].data_ptr(), L, B, s),
                ("out", [hecuda.Bfv.load(g, data, L, skip)]))
    if name.startswith("pnns_mul_transpose_vector"):
        single, m, batch = int(name[-1]), S["matrix"], 2
        v = res((batch, 2, L, n), q)
        r = m.resultCiphertextCount
        return ([v], [((batch, r, 2, 1 if single else L, n), U64)],
                lambda i, o, s: lib().hecuda_pnns_mul_transpose_vector_device(g._h, evk._h, m._h, i[0].data_ptr(), batch, single,
                                                                              o[0].data_ptr(), s),
                ("out", [m.mulTranspose(v, evk, modSwitchDownToSingle=bool(single))]))
    raise AssertionError(name)


STREAM_CASES = ["ntt_forward", "ntt_inverse", "multiply", "relinearize", "mod_switch_down", "multiply_relinearize_0",
                "multiply_relinearize_1", "apply_galois", "inner_product", "inner_product_plaintexts_all",
                "inner_product_plaintexts_mask", "plaintext_to_eval", "poly_add", "poly_sub", "poly_mul", "poly_neg",
                "poly_mul_scalars", "poly_serialize", "poly_load", "pnns_mul_transpose_vector_0",
                "pnns_mul_transpose_vector_1"]


@pytest.mark.parametrize("name", STREAM_CASES)
def test_device_call_runs_on_the_callers_stream_without_synchronising(small, name):
    """Enqueued behind the caller's (sleeping) stream, on that stream only, and equal to the host-pointer call."""
    inputs, outputs, call, (where, want) = _stream_case(name, small)
    got_in, got_out = run_on_busy_stream(inputs, outputs, call)
    got = got_in if where == "in" else got_out
    for k, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a.reshape(b.shape), b), f"{name}: {where}put {k} differs from the host-pointer call"


def test_concurrent_callers_on_one_context_and_key():
    """Four host threads, each on its own stream, multiply and relinearize different batches at once."""
    n = STREAM_N
    moduli = orc.generate_primes([55] * 4, False, n)
    t = 65537
    g = make_context(n, moduli, t, chunk=STREAM_CHUNK)
    L, K, B, rounds = g.L, g.L + 1, STREAM_BATCH, 3
    gen = generator(107)
    key = host(uniform(gen, (L, 2, K, n), moduli))
    evk = hecuda.EvaluationKey(g, key)
    inputs = [[(uniform(gen, (B, 2, L, n), moduli[:L]), uniform(gen, (B, 2, L, n), moduli[:L])) for _ in range(rounds)]
              for _ in range(4)]
    torch.cuda.synchronize()
    results, errors = {}, []
    start = threading.Barrier(4)

    def worker(tid):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                outs = []
                start.wait()
                for a, b in inputs[tid]:
                    prod = torch.empty((B, 3, L, n), dtype=torch.int64, device="cuda")
                    relin = torch.empty((B, 2, L, n), dtype=torch.int64, device="cuda")
                    ok(lib().hecuda_bfv_multiply_device(g._h, a.data_ptr(), b.data_ptr(), prod.data_ptr(), B, s.cuda_stream))
                    ok(lib().hecuda_bfv_relinearize_device(g._h, evk._h, prod.data_ptr(), L, relin.data_ptr(), B, s.cuda_stream))
                    outs.append((prod, relin))
            s.synchronize()
            results[tid] = [(host(p), host(r)) for p, r in outs]
        except Exception as exc:  # noqa: BLE001
            errors.append(exc)

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    o = orc.Context(n, moduli, t)
    for tid in range(4):
        for k, (a, b) in enumerate(inputs[tid]):
            want_prod = o.mul(host(a), host(b))
            assert np.array_equal(results[tid][k][0], want_prod), (tid, k)
            assert np.array_equal(results[tid][k][1], o.relinearize(want_prod, key)), (tid, k)
    evk.close()
    g.close()


# ================================================================================ C. graph capture
def capture(call):
    """Warm up once, then capture `call(stream)` into a CUDA graph."""
    ok(call(stream_ptr()))
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ok(call(stream_ptr()))
    return graph


@pytest.mark.parametrize("n", [8192, 16384])
def test_graph_captured_ntt_forward(n):
    moduli = orc.generate_primes([55] * 4, False, n)
    g = make_context(n, moduli, 65537)
    L, polys = g.L, 6
    buf = torch.zeros((polys, L, n), dtype=torch.int64, device="cuda")
    graph = capture(lambda s: lib().hecuda_ntt_forward_device(g._h, hecuda.BASE_Q, buf.data_ptr(), L, polys, s))
    for seed in (1, 2):
        x = uniform(generator(200 + seed), (polys, L, n), moduli[:L])
        buf.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(host(buf).reshape(-1, n), orc.ntt_forward(n, moduli[:L], host(x))), seed
    del graph
    g.close()


def test_graph_captured_multiply():
    n, moduli, t, _ = bench.workload_params("C2")
    g = make_context(n, moduli, t, chunk=3)
    L, B = g.L, 5  # chunks of 3 and 2
    lhs, rhs = (torch.zeros((B, 2, L, n), dtype=torch.int64, device="cuda") for _ in range(2))
    out = torch.zeros((B, 3, L, n), dtype=torch.int64, device="cuda")
    graph = capture(lambda s: lib().hecuda_bfv_multiply_device(g._h, lhs.data_ptr(), rhs.data_ptr(), out.data_ptr(), B, s))
    o = orc.Context(n, moduli, t)
    for seed in (1, 2):
        gen = generator(210 + seed)
        lhs.copy_(uniform(gen, (B, 2, L, n), moduli[:L]))
        rhs.copy_(uniform(gen, (B, 2, L, n), moduli[:L]))
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(host(out), o.mul(host(lhs), host(rhs))), seed
    del graph
    g.close()


def test_graph_captured_c3_step():
    n, moduli, t, _ = bench.workload_params("C3")
    g = make_context(n, moduli, t, chunk=2)
    L, K, B = g.L, g.L + 1, 3
    key = host(uniform(generator(220), (L, 2, K, n), moduli))
    evk = hecuda.EvaluationKey(g, key)
    ct3 = torch.zeros((B, 3, L, n), dtype=torch.int64, device="cuda")
    relin = torch.zeros((B, 2, L, n), dtype=torch.int64, device="cuda")
    down = torch.zeros((B, 2, L - 1, n), dtype=torch.int64, device="cuda")

    def step(s):
        rc = lib().hecuda_bfv_relinearize_device(g._h, evk._h, ct3.data_ptr(), L, relin.data_ptr(), B, s)
        return rc or lib().hecuda_bfv_mod_switch_down_device(g._h, relin.data_ptr(), 2, L, down.data_ptr(), B, s)

    graph = capture(step)
    o = orc.Context(n, moduli, t)
    for seed in (1, 2):
        ct3.copy_(uniform(generator(220 + seed), (B, 3, L, n), moduli[:L]))
        graph.replay()
        torch.cuda.synchronize()
        want = o.relinearize(host(ct3), key)
        assert np.array_equal(host(relin), want), seed
        assert np.array_equal(host(down), o.mod_switch_down(want)), seed
    del graph
    evk.close()
    g.close()


@pytest.mark.parametrize("mod_switch", [0, 1])
def test_graph_captured_multiply_relinearize(mod_switch):
    n, moduli, t, _ = bench.workload_params("C2")
    g = make_context(n, moduli, t, chunk=4)
    L, K, B = g.L, g.L + 1, 5  # chunks of 2, 2 and 1
    key = host(uniform(generator(230), (L, 2, K, n), moduli))
    evk = hecuda.EvaluationKey(g, key)
    lhs, rhs = (torch.zeros((B, 2, L, n), dtype=torch.int64, device="cuda") for _ in range(2))
    out = torch.zeros((B, 2, L - mod_switch, n), dtype=torch.int64, device="cuda")
    graph = capture(lambda s: lib().hecuda_bfv_multiply_relinearize_device(g._h, evk._h, lhs.data_ptr(), rhs.data_ptr(),
                                                                           mod_switch, out.data_ptr(), B, s))
    o = orc.Context(n, moduli, t)
    for seed in (1, 2):
        gen = generator(230 + seed)
        lhs.copy_(uniform(gen, (B, 2, L, n), moduli[:L]))
        rhs.copy_(uniform(gen, (B, 2, L, n), moduli[:L]))
        graph.replay()
        torch.cuda.synchronize()
        want = o.relinearize(o.mul(host(lhs), host(rhs)), key)
        assert np.array_equal(host(out), o.mod_switch_down(want) if mod_switch else want), seed
    del graph
    evk.close()
    g.close()


# ================================================================================ D. N = 2^15 past 65535 polynomials
def test_ntt_2_15_past_65535_polynomials():
    """65537 one-row polynomials at N = 2^15 (16 GiB): 8 distinct rows tiled, checked on the device against the oracle's
    transforms of those rows; the inverse must restore them (the merge kernel past 65535 polynomials)."""
    n, polys, distinct = 1 << 15, 65537, 8
    require_free(polys * n * 8 + 2 * GiB, "65537 polynomials at N = 2^15")
    moduli = orc.generate_primes([55, 55], False, n)
    g = make_context(n, moduli, 65537)
    base = uniform(generator(300), (distinct, 1, n), moduli[:1]).view(distinct, n)
    want = torch.from_numpy(orc.ntt_forward(n, moduli[:1], host(base)).view(np.int64)).cuda()
    data = torch.empty((polys, n), dtype=torch.int64, device="cuda")
    for k in range(distinct):
        data[k::distinct] = base[k]
    ok(lib().hecuda_ntt_forward_device(g._h, hecuda.BASE_Q, data.data_ptr(), 1, polys, stream_ptr()))
    for k in range(distinct):
        assert bool((data[k::distinct] == want[k]).all()), f"forward: rows {k} mod {distinct} differ"
    ok(lib().hecuda_ntt_inverse_device(g._h, hecuda.BASE_Q, data.data_ptr(), 1, polys, stream_ptr()))
    for k in range(distinct):
        assert bool((data[k::distinct] == base[k]).all()), f"inverse: rows {k} mod {distinct} differ"
    del data
    g.close()


# ================================================================================ E. the argument contract
def test_device_argument_contract(small):
    """Empty batches return HECUDA_OK without launching; NULL buffers, foreign and missing keys and a modulus switch
    below two moduli are refused, as by the host variants, before anything is enqueued."""
    S = small
    g, n, L, evk, m, e = S["g"], S["n"], S["L"], S["evk"], S["matrix"], S["element"]
    moduli, Q = S["moduli"], hecuda.BASE_Q
    other = make_context(n, moduli, S["t"])
    foreign = hecuda.EvaluationKey(other, S["residues"]((L, 2, L + 1, n), moduli))
    foreign.setGaloisKey(e, S["residues"]((L, 2, L + 1, n), moduli))
    bare = hecuda.EvaluationKey(g, None)  # neither a relinearization key nor Galois keys
    buf = torch.zeros((4, 3, L, n), dtype=torch.int64, device="cuda")
    p = buf.data_ptr()
    scalars = np.ones(L, dtype=np.uint64)
    torch.cuda.synchronize()
    f = lib()
    before = hecuda.kernel_launch_count()

    def calls(x, count):
        """Every device entry point with all its buffers x and count items."""
        s = stream_ptr()
        return {
            "ntt_forward": f.hecuda_ntt_forward_device(g._h, Q, x, L, count, s),
            "ntt_inverse": f.hecuda_ntt_inverse_device(g._h, Q, x, L, count, s),
            "multiply": f.hecuda_bfv_multiply_device(g._h, x, x, x, count, s),
            "relinearize": f.hecuda_bfv_relinearize_device(g._h, evk._h, x, L, x, count, s),
            "mod_switch_down": f.hecuda_bfv_mod_switch_down_device(g._h, x, 2, L, x, count, s),
            "multiply_relinearize": f.hecuda_bfv_multiply_relinearize_device(g._h, evk._h, x, x, 1, x, count, s),
            "apply_galois": f.hecuda_bfv_apply_galois_device(g._h, evk._h, x, L, e, x, count, s),
            "inner_product": f.hecuda_bfv_inner_product_device(g._h, x, x, x, 2, count, s),
            "inner_product_plaintexts": f.hecuda_bfv_inner_product_plaintexts_device(g._h, x, 2, L, 2, x, None, x, count, s),
            "plaintext_to_eval": f.hecuda_plaintext_to_eval_device(g._h, x, L, x, count, s),
            "poly_add": f.hecuda_poly_add_device(g._h, Q, x, x, L, count, s),
            "poly_sub": f.hecuda_poly_sub_device(g._h, Q, x, x, L, count, s),
            "poly_mul": f.hecuda_poly_mul_device(g._h, Q, x, x, L, count, s),
            "poly_neg": f.hecuda_poly_neg_device(g._h, Q, x, L, count, s),
            "poly_mul_scalars": f.hecuda_poly_mul_scalars_device(g._h, Q, x, scalars.ctypes.data, L, count, s),
            "poly_serialize": f.hecuda_poly_serialize_device(g._h, Q, x, 0, x, L, count, s),
            "poly_load": f.hecuda_poly_load_device(g._h, Q, x, 0, x, L, count, s),
            "pnns_mul_transpose_vector": f.hecuda_pnns_mul_transpose_vector_device(g._h, evk._h, m._h, x, count, 1, x, s),
        }

    for x in (None, p):
        rcs = calls(x, 0)
        assert all(rc == OK for rc in rcs.values()), {k: v for k, v in rcs.items() if v != OK}
    rcs = calls(None, 2)
    assert all(rc == ERR_INVALID_ARGUMENT for rc in rcs.values()), {k: v for k, v in rcs.items() if v != ERR_INVALID_ARGUMENT}
    assert f.hecuda_bfv_mod_switch_down_device(g._h, p, 2, 1, p, 2, stream_ptr()) == ERR_INVALID_ARGUMENT

    # keys: the device variants give the host variants' codes
    hb = np.zeros((4, 3, L, n), dtype=np.uint64)
    hp = hb.ctypes.data
    s = stream_ptr()
    keyed = {  # (device call, host call)
        "relinearize": (lambda k: f.hecuda_bfv_relinearize_device(g._h, k._h, p, L, p, 2, s),
                        lambda k: f.hecuda_bfv_relinearize(g._h, k._h, hp, L, hp, 2)),
        "multiply_relinearize": (lambda k: f.hecuda_bfv_multiply_relinearize_device(g._h, k._h, p, p, 1, p, 2, s),
                                 lambda k: f.hecuda_bfv_multiply_relinearize(g._h, k._h, hp, hp, 1, hp, 2)),
        "apply_galois": (lambda k: f.hecuda_bfv_apply_galois_device(g._h, k._h, p, L, e, p, 2, s),
                         lambda k: f.hecuda_bfv_apply_galois(g._h, k._h, hp, L, e, hp, 2)),
        "pnns_mul_transpose_vector": (lambda k: f.hecuda_pnns_mul_transpose_vector_device(g._h, k._h, m._h, p, 2, 1, p, s),
                                      lambda k: f.hecuda_pnns_mul_transpose_vector(g._h, k._h, m._h, hp, 2, 1, hp)),
    }
    for key, code in ((foreign, ERR_INVALID_ARGUMENT), (bare, ERR_MISSING_KEY)):
        for name, (on_device, on_host) in keyed.items():
            got, want = on_device(key), on_host(key)
            assert got == want == code, (name, got, want, code)
    torch.cuda.synchronize()
    assert hecuda.kernel_launch_count() == before
    foreign.close()
    bare.close()
    other.close()
