"""Every batched C-ABI operation three ways: hecuda_X on uint64 host buffers, hecuda_X_device on device buffers and
hecuda_u32_X on uint32 host buffers.  All three run one description of the operation (csrc/capi.cu), so:

A. they give identical words, at N = 4096 on a 64-bit and a 32-bit context, with HECUDA_CHUNK=3 and batches of 1, 7
   and 70: ragged device chunks and multi-stage host pipelines with tail stages, on one and on two staged inputs;
B. each call launches what its chunk schedule gives: a device call ceil(batch / items per launch) times the launches of
   a one-item call, a host call that many per pipeline stage, plus one widen per staged input and one narrow per stage
   on uint32 buffers.  Items per launch and the stage hints restate the library's rules; the stage count follows the
   host pipeline's clamp;
C. a refused argument gives the same code and message through every flavour and launches nothing."""
import contextlib
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import hecuda  # noqa: E402
from hecuda import pnns  # noqa: E402
from oracle import oracle as orc  # noqa: E402

N = 4096
CHUNK = 3  # HECUDA_CHUNK, i.e. h->chunk
BATCHES = [1, 7, 70]
T = 65537  # prime = 1 mod 2N: SIMD encoding
STAGE = 4 << 20  # words: the stage budget of the operations not sized by h->chunk
SIMD_PER_LAUNCH = (1 << 25) // N
WHOLE = 1 << 62  # one device launch for the whole batch
OK, ERR_INVALID_ARGUMENT, ERR_MISSING_KEY = 0, -1, -5


def lib():
    return hecuda.load_library()


def last_error():
    return (lib().hecuda_last_error() or b"").decode()


@contextlib.contextmanager
def chunk_env(chunk):
    old = os.environ.get("HECUDA_CHUNK")
    os.environ["HECUDA_CHUNK"] = str(chunk)
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("HECUDA_CHUNK", None)
        else:
            os.environ["HECUDA_CHUNK"] = old


def stages(batch, hint):
    """Host pipeline stages: items per stage max(1, min(hint, batch)), from 64 items on at most max(16, ceil(batch / 16))."""
    chunk = max(1, min(hint, batch))
    if batch >= 64:
        chunk = min(chunk, max(16, -(-batch // 16)))
    return -(-batch // chunk)


def entry_point(name, flavour):
    return getattr(lib(), ("hecuda_u32_" if flavour == "u32" else "hecuda_") + name + ("_device" if flavour == "device" else ""))


def make_context(moduli, word32):
    with chunk_env(CHUNK):
        return hecuda.Context(N, moduli, T, scalar=np.uint32 if word32 else np.uint64)


@pytest.fixture(scope="module", params=["word64", "word32"])
def ctx(request):
    word32 = request.param == "word32"
    moduli = orc.generate_primes([28, 28, 29] if word32 else [55] * 4, False, N)
    g = make_context(moduli, word32)
    L, K = g.L, g.L + 1
    rng = np.random.default_rng(11)

    def residues(shape, mods):
        q = np.array(mods, dtype=np.uint64).reshape(len(mods), 1)
        return (rng.integers(0, 1 << 62, size=shape, dtype=np.uint64) % q).astype(np.uint64)

    evk = hecuda.EvaluationKey(g, residues((L, 2, K, N), moduli))
    element = pnns.GaloisElement.rotatingColumns(-1, N)
    evk.setGaloisKey(element, residues((L, 2, K, N), moduli))
    yield dict(g=g, word32=word32, moduli=moduli, L=L, evk=evk, element=element, residues=residues, rng=rng)
    evk.close()
    g.close()


class Op:
    """One batched operation at one batch size: `args(inputs, out, shared)` gives the arguments after the context handle
    (and before the device flavour's stream), the same for every flavour."""

    def __init__(self, label, name, inputs, out_shape, args, per_launch, hint, shared=(), flavours=("host", "device", "u32"),
                 in_place=False):
        self.label, self.name, self.inputs, self.out_shape, self.args = label, name, inputs, out_shape, args
        self.per_launch, self.hint, self.shared, self.flavours, self.in_place = per_launch, hint, shared, flavours, in_place


def operations(S, B):
    L, evk, e, rng, res = S["L"], S["evk"]._h, S["element"], S["rng"], S["residues"]
    q = S["moduli"][:L]
    Q, rows_qbsk = hecuda.BASE_Q, 2 * L + 1
    pairs, terms, values = 2, 3, N // 2
    ct = lambda polys: res((B, polys, L, N), q)  # noqa: E731
    plain = lambda shape: rng.integers(0, T, size=shape, dtype=np.uint64)  # noqa: E731
    ops = [
        Op("ntt_forward", "ntt_forward", [res((B, L, N), q)], None, lambda i, o, s: (Q, i[0], L, B), WHOLE, STAGE // (L * N),
           in_place=True),
        Op("ntt_inverse", "ntt_inverse", [res((B, L, N), q)], None, lambda i, o, s: (Q, i[0], L, B), WHOLE, STAGE // (L * N),
           in_place=True),
        Op("multiply", "bfv_multiply", [ct(2), ct(2)], (B, 3, L, N), lambda i, o, s: (i[0], i[1], o, B), CHUNK, CHUNK),
        Op("relinearize", "bfv_relinearize", [ct(3)], (B, 2, L, N), lambda i, o, s: (evk, i[0], L, o, B), CHUNK, CHUNK),
        Op("mod_switch_down", "bfv_mod_switch_down", [ct(2)], (B, 2, L - 1, N), lambda i, o, s: (i[0], 2, L, o, B), WHOLE,
           STAGE // (2 * L * N)),
        Op("relinearize_mod_switch_down", "bfv_relinearize_mod_switch_down", [ct(3)], (B, 2, L - 1, N),
           lambda i, o, s: (evk, i[0], L, o, B), None, CHUNK, flavours=("host", "u32")),
        Op("apply_galois", "bfv_apply_galois", [ct(2)], (B, 2, L, N), lambda i, o, s: (evk, i[0], L, e, o, B), CHUNK, CHUNK),
        Op("inner_product", "bfv_inner_product", [res((B, pairs, 2, L, N), q), res((B, pairs, 2, L, N), q)], (B, 3, L, N),
           lambda i, o, s: (i[0], i[1], o, pairs, B), max(1, CHUNK // pairs), max(1, CHUNK // pairs)),
        Op("encode_simd", "bfv_encode_simd", [plain((B, values))], (B, L, N), lambda i, o, s: (i[0], values, L, o, B),
           SIMD_PER_LAUNCH, STAGE // (L * N)),
        Op("decode_simd", "bfv_decode_simd", [res((B, L, N), q)], (B, N), lambda i, o, s: (i[0], L, o, B), SIMD_PER_LAUNCH,
           STAGE // (L * N)),
        # one plaintext for the whole batch is uploaded once, outside the pipeline: one staged input
        Op("translate_broadcast", "bfv_plaintext_translate", [ct(2)], (B, 2, L, N),
           lambda i, o, s: (i[0], 2, L, s[0], 1, hecuda.PLAINTEXT_ADD, o, B), WHOLE, STAGE // (2 * L * N),
           shared=[plain((1, N))]),
        Op("lift_q_to_qbsk", "rnstool_lift_q_to_qbsk", [res((B, L, N), q)], (B, rows_qbsk, N), lambda i, o, s: (i[0], o, B),
           None, STAGE // (rows_qbsk * N), flavours=("host", "u32")),
        Op("floor_qbsk_to_q", "rnstool_floor_qbsk_to_q", [res((B, rows_qbsk, N), [min(q)] * rows_qbsk)], (B, L, N),
           lambda i, o, s: (i[0], o, B), None, STAGE // (rows_qbsk * N), flavours=("host", "u32")),
        Op("plaintext_to_eval", "plaintext_to_eval", [plain((B, N))], (B, L, N), lambda i, o, s: (i[0], L, o, B), WHOLE,
           STAGE // (L * N), flavours=("host", "device")),
        # the query ciphertexts are shared by every output row
        Op("inner_product_plaintexts", "bfv_inner_product_plaintexts", [res((B, terms, L, N), q)], (B, 2, L, N),
           lambda i, o, s: (s[0], 2, L, terms, i[0], None, o, B), WHOLE, (32 << 20) // (terms * L * N),
           shared=[res((terms, 2, L, N), q)], flavours=("host", "device")),
        Op("ntt_forward_rows", "ntt_forward_rows", [res((B, 1, N), q[:1])], None, lambda i, o, s: (q[0], i[0], B), None,
           STAGE // N, flavours=("host",), in_place=True),
        Op("poly_apply_galois", "poly_apply_galois", [res((B, L, N), q)], (B, L, N), lambda i, o, s: (Q, 0, i[0], o, L, B, e),
           None, STAGE // (L * N), flavours=("host",)),
        Op("poly_multiply_power_of_x", "poly_multiply_power_of_x", [res((B, L, N), q)], (B, L, N),
           lambda i, o, s: (Q, i[0], o, L, B, 5), None, STAGE // (L * N), flavours=("host",)),
    ]
    for m in (0, 1):
        ops.append(Op(f"multiply_relinearize_{m}", "bfv_multiply_relinearize", [ct(2), ct(2)], (B, 2, L - m, N),
                      lambda i, o, s, m=m: (evk, i[0], i[1], m, o, B), max(1, CHUNK // 2), max(1, CHUNK // 2)))
    # one plaintext per ciphertext: two staged inputs (at B = 1, plaintext_count = 1 makes it the broadcast)
    ops.append(Op("translate", "bfv_plaintext_translate", [ct(2), plain((B, N))], (B, 2, L, N),
                  lambda i, o, s: (i[0], 2, L, i[1], B, hecuda.PLAINTEXT_SUB, o, B), WHOLE, STAGE // (2 * L * N)))
    return ops


def run(S, op, flavour):
    """One flavour of `op`: (rc, kernel launches, output words as uint64)."""
    fn = entry_point(op.name, flavour)
    if flavour == "device":
        ins = [torch.from_numpy(a.view(np.int64)).cuda() for a in op.inputs]
        shared = [torch.from_numpy(a.view(np.int64)).cuda() for a in op.shared]
        out = torch.zeros(op.out_shape, dtype=torch.int64, device="cuda") if op.out_shape else None
        args = op.args([t.data_ptr() for t in ins], out.data_ptr() if out is not None else None, [t.data_ptr() for t in shared])
        args += (torch.cuda.current_stream().cuda_stream,)
    else:
        dtype = np.uint32 if flavour == "u32" else np.uint64
        ins = [np.ascontiguousarray(a.astype(dtype)) for a in op.inputs]
        shared = [np.ascontiguousarray(a.astype(dtype)) for a in op.shared]
        out = np.zeros(op.out_shape, dtype) if op.out_shape else None
        args = op.args([a.ctypes.data for a in ins], out.ctypes.data if out is not None else None, [a.ctypes.data for a in shared])
    torch.cuda.synchronize()
    before = hecuda.kernel_launch_count()
    rc = fn(S["g"]._h, *args)
    torch.cuda.synchronize()
    launches = hecuda.kernel_launch_count() - before
    got = ins[0] if op.in_place else out
    got = got.cpu().numpy().view(np.uint64) if flavour == "device" else got.astype(np.uint64)
    return rc, launches, got


# ================================================================================ A, B
@pytest.mark.parametrize("batch", BATCHES)
def test_flavours_agree_and_follow_the_chunk_schedule(ctx, batch):
    S = ctx
    flavours_here = lambda op: [f for f in op.flavours if f != "u32" or S["word32"]]  # noqa: E731
    one = {}  # launches of a one-item call
    for op in operations(S, 1):
        for flavour in flavours_here(op):
            if flavour != "u32":
                rc, one[op.label, flavour], _ = run(S, op, flavour)
                assert rc == OK, (op.label, flavour, rc, last_error())
    failures = []
    for op in operations(S, batch):
        if op.label == "translate" and batch == 1:
            continue
        base = one[op.label, "host"]
        results = {}
        for flavour in flavours_here(op):
            tag = f"{op.label} ({flavour}, batch {batch})"
            rc, launches, got = run(S, op, flavour)
            if rc != OK:
                failures.append(f"{tag}: rc {rc}: {last_error()}")
                continue
            if flavour == "device":
                if one[op.label, "device"] != base:
                    failures.append(f"{tag}: a one-item call launches {one[op.label, 'device']}, the host's {base}")
                want = -(-batch // min(op.per_launch, batch)) * base
            else:
                want = stages(batch, op.hint) * (base + (len(op.inputs) + 1 if flavour == "u32" else 0))
            if launches != want:
                failures.append(f"{tag}: {launches} launches, the schedule gives {want}")
            results[flavour] = got
        for flavour, got in results.items():
            if "host" in results and not np.array_equal(got, results["host"]):
                failures.append(f"{op.label} (batch {batch}): the {flavour} call differs from the uint64 host call")
    assert not failures, "\n".join(failures)


# ================================================================================ C
def test_refusals_agree_and_launch_nothing(ctx):
    """A foreign key, a missing relinearization or Galois key, moduli_count out of range and NULL buffers: the same code
    and message from every flavour, and no kernel launched."""
    S = ctx
    g, L, moduli, e, evk = S["g"], S["L"], S["moduli"], S["element"], S["evk"]._h
    other = make_context(moduli, S["word32"])
    foreign = hecuda.EvaluationKey(other, S["residues"]((L, 2, L + 1, N), moduli))
    foreign.setGaloisKey(e, S["residues"]((L, 2, L + 1, N), moduli))
    bare = hecuda.EvaluationKey(g, None)  # neither a relinearization key nor Galois keys
    B, add = 2, hecuda.PLAINTEXT_ADD
    unkeyed = next(x for x in (5, 2 * N - 1) if x != e)  # a valid Galois element the key has no key for
    cases = []  # (label, entry point, arguments given the flavour's buffer p, expected code)
    for key_label, key, code in (("foreign key", foreign._h, ERR_INVALID_ARGUMENT), ("missing key", bare._h, ERR_MISSING_KEY)):
        cases += [
            (f"relinearize, {key_label}", "bfv_relinearize", lambda p, k=key: (k, p, L, p, B), code),
            (f"relinearize_mod_switch_down, {key_label}", "bfv_relinearize_mod_switch_down", lambda p, k=key: (k, p, L, p, B), code),
            (f"multiply_relinearize, {key_label}", "bfv_multiply_relinearize", lambda p, k=key: (k, p, p, 1, p, B), code),
            (f"apply_galois, {key_label}", "bfv_apply_galois", lambda p, k=key: (k, p, L, e, p, B), code),
        ]
    cases += [
        ("apply_galois, element without a key", "bfv_apply_galois", lambda p: (evk, p, L, unkeyed, p, B), ERR_MISSING_KEY),
        ("relinearize, moduli_count 0", "bfv_relinearize", lambda p: (evk, p, 0, p, B), ERR_INVALID_ARGUMENT),
        ("apply_galois, moduli_count L + 1", "bfv_apply_galois", lambda p: (evk, p, L + 1, e, p, B), ERR_INVALID_ARGUMENT),
        ("mod_switch_down, moduli_count 1", "bfv_mod_switch_down", lambda p: (p, 2, 1, p, B), ERR_INVALID_ARGUMENT),
        ("multiply, NULL out", "bfv_multiply", lambda p: (p, p, None, B), ERR_INVALID_ARGUMENT),
        ("relinearize, NULL input", "bfv_relinearize", lambda p: (evk, None, L, p, B), ERR_INVALID_ARGUMENT),
        ("inner_product, NULL rhs", "bfv_inner_product", lambda p: (p, None, p, 2, B), ERR_INVALID_ARGUMENT),
        ("encode_simd, NULL out", "bfv_encode_simd", lambda p: (p, 4, L, None, B), ERR_INVALID_ARGUMENT),
        ("decode_simd, NULL input", "bfv_decode_simd", lambda p: (None, L, p, B), ERR_INVALID_ARGUMENT),
        ("plaintext_translate, NULL plaintext", "bfv_plaintext_translate", lambda p: (p, 2, L, None, 1, add, p, B),
         ERR_INVALID_ARGUMENT),
        ("ntt_forward, NULL data", "ntt_forward", lambda p: (hecuda.BASE_Q, None, L, B), ERR_INVALID_ARGUMENT),
    ]
    dbuf = torch.zeros((B, 3, L, N), dtype=torch.int64, device="cuda")
    hbuf = np.zeros((B, 3, L, N), dtype=np.uint64)
    stream = torch.cuda.current_stream().cuda_stream
    failures = []
    torch.cuda.synchronize()
    before = hecuda.kernel_launch_count()
    for label, name, args, code in cases:
        seen = {}
        for flavour in ("host", "device", "u32"):
            if flavour == "u32" and not S["word32"]:
                continue
            try:
                fn = entry_point(name, flavour)
            except AttributeError:  # host-only operations
                continue
            if flavour == "device":
                rc = fn(g._h, *args(dbuf.data_ptr()), stream)
            else:
                rc = fn(g._h, *args(hbuf.ctypes.data))
            seen[flavour] = (rc, last_error())
        if len(set(seen.values())) != 1 or next(iter(seen.values()))[0] != code:
            failures.append(f"{label}: {seen}, expected code {code}")
    torch.cuda.synchronize()
    launched = hecuda.kernel_launch_count() - before
    foreign.close()
    bare.close()
    other.close()
    assert not failures, "\n".join(failures)
    assert launched == 0, f"refused calls launched {launched} kernels"
