"""Many clients' seeded evaluation keys in one call (hecuda_evk_create_serialized_many, EvaluationKey.fromSerializedMany).
Every key must equal, word for word, the same client's key from hecuda_evk_create_serialized (and a sample the
oracle's expansion), serve the many-clients MulPir and PNNS calls like singly loaded keys, cost 1 + ceil(K / GROUP)
launches per call, live and die independently of the other keys of its call, and be refused exactly like the single
call."""
import ctypes as C
import math
import random
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import evk_wire_ref as ref
import hecuda
from hecuda import pir, pnns
from oracle import oracle as orc
from oracle import pir_oracle as opir
from rlwe_shapes import read_device
from test_gpu_evk_wire import (ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED, KEY_SETS, PIR_MODULI, TEST_MODULI_BITS, check_wire,
                               contexts, seeded_keys)
from test_gpu_pir_clients import Setup
from test_gpu_pnns_clients import Server

GROUP = 16  # HECUDA_EVK_LOAD_GROUP
COUNTS = [1, 2, GROUP, GROUP + 1, 4 * GROUP + 3]
CONFIGS = {"relin_galois": (True, 2), "galois_only": (False, 2), "relin_only": (True, 0)}


def lib():
    return hecuda.load_library()


class Wire:
    """Clients' seeded keys of one config as raw bytes: per client one poly0 buffer (C x B) and one seed buffer
    (C x 32), the relinearization key first and then `elements` in order.  poly0 is the serialization of uniform
    residues below every key-switching modulus, so every buffer is a valid key on the wire."""

    def __init__(self, n, moduli, t, relin, elements, count, seed):
        self.n, self.moduli, self.relin, self.elements = n, moduli, relin, np.ascontiguousarray(elements, dtype=np.uint32)
        ser = hecuda.Context(n, moduli, t)  # a UInt32 context takes the same bytes
        self.L = ser.L
        self.cts = (int(relin) + len(elements)) * self.L
        self.B = hecuda.Bfv.serializationByteCount(ser, self.L + 1, base=hecuda.BASE_KEYSWITCH)
        rng = np.random.default_rng(seed)
        self.poly0, self.seeds = [], []
        for _ in range(count):
            words = np.empty((self.cts, self.L + 1, n), dtype=np.uint64)
            for i, q in enumerate(moduli):
                words[:, i, :] = rng.integers(0, q, size=(self.cts, n), dtype=np.uint64)
            p = hecuda.Bfv.serialize(ser, words, base=hecuda.BASE_KEYSWITCH) if self.cts else np.zeros((0, self.B), np.uint8)
            self.poly0.append(np.ascontiguousarray(p, dtype=np.uint8).reshape(self.cts, self.B))
            self.seeds.append(ref.random_seeds(rng, self.cts))
        ser.close()

    def many(self, g, first=0, count=None):
        """hecuda_evk_create_serialized_many over clients [first, first + count): (rc, handles)."""
        count = len(self.poly0) - first if count is None else count
        out = (C.c_void_p * count)(*([1] * count))  # not NULL on entry: a failed call must leave NULL behind
        sel = range(first, first + count)
        rc = lib().hecuda_evk_create_serialized_many(
            g._h, count, int(self.relin), self.elements.ctypes.data if len(self.elements) else None, len(self.elements),
            (C.c_void_p * count)(*[self.poly0[j].ctypes.data for j in sel]),
            (C.c_void_p * count)(*[self.seeds[j].ctypes.data for j in sel]), out)
        return rc, list(out)

    def single(self, g, j):
        L, h = self.L, C.c_void_p(1)
        p, s = self.poly0[j], self.seeds[j]
        r = L if self.relin else 0
        ptr = lambda a: a.ctypes.data if a.size else None  # noqa: E731
        rc = lib().hecuda_evk_create_serialized(
            g._h, ptr(p[:r]) if self.relin else None, ptr(s[:r]) if self.relin else None,
            self.elements.ctypes.data if len(self.elements) else None, len(self.elements),
            ptr(p[r:]) if len(self.elements) else None, ptr(s[r:]) if len(self.elements) else None, C.byref(h))
        assert rc == 0, lib().hecuda_last_error()
        return h.value

    def buffers(self, handle):
        """The key's relinearization buffer (always allocated) and its Galois buffers, as words."""
        h = C.c_void_p(handle)
        p, nbytes = C.c_void_p(), C.c_uint64()
        assert lib().hecuda_evk_device_buffer(h, C.byref(p), C.byref(nbytes)) == 0
        out = [read_device(p.value, nbytes.value)] if self.relin else []
        assert nbytes.value == self.L * 2 * (self.L + 1) * self.n * 8  # L x 2 x K x N even without a relinearization key
        for e in self.elements:
            assert lib().hecuda_evk_galois_device_buffer(h, int(e), C.byref(p), C.byref(nbytes)) == 0
            out.append(read_device(p.value, nbytes.value))
        return out

    def python_forms(self):
        """The clients as EvaluationKey.generate(..., wire=True) forms."""
        L, r = self.L, (self.L if self.relin else 0)
        return [{"relinPoly0": p[:L] if self.relin else None, "relinSeeds": s[:L] if self.relin else None,
                 "galois": {int(e): (p[r + i * L:r + (i + 1) * L], s[r + i * L:r + (i + 1) * L])
                            for i, e in enumerate(self.elements)}}
                for p, s in zip(self.poly0, self.seeds)]


def destroy(handles):
    for h in handles:
        lib().hecuda_evk_destroy(C.c_void_p(h))


# ---------------------------------------------------------------- 1. bit-exact keys
@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("count", COUNTS)
@pytest.mark.parametrize("n,bits,t,word_bits", KEY_SETS)
def test_keys_equal_single_loads(n, bits, t, word_bits, count, config):
    moduli = PIR_MODULI if word_bits == 32 else orc.generate_primes(bits, False, n)
    g = hecuda.Context(n, moduli, t, scalar=np.uint32 if word_bits == 32 else np.uint64)
    relin, elements = CONFIGS[config]
    w = Wire(n, moduli, t, relin, [3, 2 * n - 1][:elements], count, seed=n + count + word_bits)
    before = hecuda.kernel_launch_count()
    rc, handles = w.many(g)
    assert rc == 0, lib().hecuda_last_error()
    assert hecuda.kernel_launch_count() - before == 1 + math.ceil(count / GROUP)
    for j, h in enumerate(handles):
        one = w.single(g, j)
        for a, b in zip(w.buffers(h), w.buffers(one)):
            assert np.array_equal(a, b), j
        destroy([one])
    # a sample against the oracle: the last client's last key ciphertext
    o = orc.Context(n, moduli, t, word_bits=word_bits)
    got = w.buffers(handles[-1])[-1].reshape(w.L, 2, w.L + 1, n)[-1]
    assert np.array_equal(got, ref.expand_seeded_key_ciphertext(o, w.poly0[-1][-1].tobytes(), w.seeds[-1][-1].tobytes()))
    destroy(handles)
    g.close()


@pytest.mark.parametrize("sources", ["pinned", "mixed"])
def test_pinned_client_buffers(sources):
    """Clients in their own pinned buffers (copied from directly, never in one copy with another client's buffer),
    or pinned and pageable in turn, give the keys of pageable buffers."""
    n = 4096
    g, _ = contexts(n, [27, 28, 28], 17)
    w = Wire(n, g.coefficientModuli, 17, True, [3, 5, 2 * n - 1], 2 * GROUP + 3, seed=31)
    rc, want = w.many(g)
    assert rc == 0
    pins = []
    for j, p in enumerate(w.poly0):
        if sources == "pinned" or j % 2:
            b = hecuda.PinnedBuffer(p.shape, np.uint8)
            b.array[:] = p
            pins.append(b)
            w.poly0[j] = b.array
    rc, got = w.many(g)
    assert rc == 0, lib().hecuda_last_error()
    for j, (a, b) in enumerate(zip(got, want)):
        for x, y in zip(w.buffers(a), w.buffers(b)):
            assert np.array_equal(x, y), j
    destroy(got + want)
    w.poly0 = None
    for b in pins:
        b.free()
    g.close()


def test_empty_config_makes_keys_without_launches():
    g, _ = contexts(16, TEST_MODULI_BITS, 1153)
    w = Wire(16, g.coefficientModuli, 1153, False, [], 3, seed=1)
    before = hecuda.kernel_launch_count()
    out = (C.c_void_p * 3)()
    assert lib().hecuda_evk_create_serialized_many(g._h, 3, 0, None, 0, None, None, out) == 0
    assert hecuda.kernel_launch_count() == before
    assert all(out)
    for h in out:
        w.buffers(h)  # the relinearization buffer is still L x 2 x K x N
    destroy(out)
    g.close()


# ---------------------------------------------------------------- 2. keys that work
def both_ways(g, o, clients, relin=True):
    """Each client's wire key loaded singly (fromSerialized) and in one call (fromSerializedMany)."""
    forms = [{"relinPoly0": c["relin_wire"][0] if relin else None, "relinSeeds": c["relin_wire"][1] if relin else None,
              "galois": c["galois_wire"]} for c in clients]
    singles = [hecuda.EvaluationKey.fromSerialized(g, f["relinPoly0"], f["relinSeeds"], f["galois"]) for f in forms]
    return singles, hecuda.EvaluationKey.fromSerializedMany(g, forms)


def test_batch_keys_serve_mulpir_wire():
    g, o = contexts(4096, [27, 28, 28], 17)
    s = Setup(g, o, 20000, 1, 2, 1, True, "hybridCompression", seed=4097)
    rng = np.random.default_rng(4097)
    elements = s.param.evaluationKeyConfig.galoisElements
    clients = []
    for c in range(3):
        sk, relin, relin_wire, okeys, galois_wire = seeded_keys(o, 600 + c, rng, elements, 8000 + 31 * c)
        # the Galois keys in another order for each client: the wrapper puts them into one order
        galois_wire = dict(reversed(list(galois_wire.items()))) if c % 2 else galois_wire
        indices = [s.rng.randrange(s.entries)]
        query = np.stack(opir.generate_query(o, s.oparam, indices, sk, 9100 + c))
        seeds = ref.random_seeds(rng, len(query))
        cts, poly0 = ref.reseed_query(o, sk, query, seeds)
        clients.append(dict(sk=sk, relin=relin, okeys=okeys, indices=indices, cts=cts, poly0=poly0, seeds=seeds,
                            relin_wire=relin_wire, galois_wire=galois_wire))
    singles, batch = both_ways(g, o, clients)
    poly0, seeds = np.stack([c["poly0"] for c in clients]), np.stack([c["seeds"] for c in clients])
    want, _ = pir.PirWire.computeResponses(s.server, poly0, seeds, singles)
    got, _ = pir.PirWire.computeResponses(s.server, poly0, seeds, batch)
    assert np.array_equal(got, want)
    for c, k in zip(clients, batch):
        c["key"] = k
    check_wire(s, clients, oracle_clients={0})  # single-client parity, oracle bytes, and decryption to the entries
    for k in singles:
        k.close()
    s.close(clients)
    g.close()


def test_batch_keys_serve_pnns_wire():
    s = Server(64, 65537, (55, 55, 55), 40, 12, 4, seed=77)
    o, rng = s.o, np.random.default_rng(77)
    clients = []
    for j in range(3):
        sk, _, relin_wire, okeys, wire = seeded_keys(o, 700 + j, rng, s.elements, 9000 + 31 * j)
        query, cts = s.query(700 + j, sk)
        seeds = ref.random_seeds(rng, len(cts))
        seeded, poly0 = ref.reseed_query(o, sk, cts, seeds)
        clients.append(dict(sk=sk, okeys=okeys, query=query, cts=seeded, poly0=poly0, seeds=seeds,
                            relin_wire=relin_wire, galois_wire=wire))
    singles, batch = both_ways(s.g, o, clients, relin=False)
    poly0, seeds = np.stack([c["poly0"] for c in clients]), np.stack([c["seeds"] for c in clients])
    want, skips = pnns.PnnsWire.computeResponses(s.matrix, poly0, seeds, s.dims, singles)
    got, _ = pnns.PnnsWire.computeResponses(s.matrix, poly0, seeds, s.dims, batch)
    assert np.array_equal(got, want)
    n, q0 = s.n, o.q[:1]
    half = opir.serialization_byte_count(n, q0, skips[0])
    for j, c in enumerate(clients):
        recovered = [np.stack([opir.load_poly(n, q0, got[j, i, :half].tobytes(), skips[0]),
                               opir.load_poly(n, q0, got[j, i, half:].tobytes(), skips[1])]) for i in range(got.shape[1])]
        s.assert_decrypts(c, recovered, f"client {j}")  # the distances
    for k in singles:
        k.close()
    for c, k in zip(clients, batch):
        c["key"] = k
    s.close(clients)


def test_relinearize_and_galois_match_single_keys():
    n = 2048
    g, o = contexts(n, [62, 62, 62], 65537)
    moduli, L = g.coefficientModuli, g.L
    w = Wire(n, moduli, 65537, True, [3, 2 * n - 1], GROUP + 2, seed=5)
    batch = hecuda.EvaluationKey.fromSerializedMany(g, w.python_forms())
    ct3 = orc.fill_uniform(5, moduli[:L], n, 2 * 3 * L).reshape(2, 3, L, n)
    ct = orc.fill_uniform(6, moduli[:L], n, 2 * 2 * L).reshape(2, 2, L, n)
    for j in (0, GROUP, GROUP + 1):
        single = hecuda.EvaluationKey.fromSerialized(g, **w.python_forms()[j])
        assert np.array_equal(hecuda.Bfv.relinearize(g, ct3, batch[j]), hecuda.Bfv.relinearize(g, ct3, single)), j
        for e in (3, 2 * n - 1):
            assert np.array_equal(hecuda.Bfv.applyGalois(g, ct, e, batch[j]), hecuda.Bfv.applyGalois(g, ct, e, single)), j
        single.close()
    for k in batch:
        k.close()
    g.close()


# ---------------------------------------------------------------- 4. lifetimes
def test_lifetimes():
    n = 64
    g, o = contexts(n, [55, 55, 55], 65537)
    moduli, L = g.coefficientModuli, g.L
    count = 2 * GROUP + 5
    w = Wire(n, moduli, 65537, True, [3, 2 * n - 1], count, seed=9)
    keys = hecuda.EvaluationKey.fromSerializedMany(g, w.python_forms())
    ct = orc.fill_uniform(6, moduli[:L], n, 2 * 2 * L).reshape(2, 2, L, n)
    ct3 = orc.fill_uniform(5, moduli[:L], n, 2 * 3 * L).reshape(2, 3, L, n)
    want = [hecuda.Bfv.applyGalois(g, ct, 3, k) for k in keys]
    # destroy in a shuffled order while the others keep answering
    order = list(range(count))
    random.Random(3).shuffle(order)
    alive = set(order)
    for step, j in enumerate(order[: count - 4]):
        keys[j].close()
        alive.discard(j)
        if step % 5 == 0:
            for i in alive:
                assert np.array_equal(hecuda.Bfv.applyGalois(g, ct, 3, keys[i]), want[i]), (step, i)
    rest = sorted(alive)
    # setGaloisKey replaces a key inside a batch-loaded handle, which is then destroyed
    replaced = keys[rest[0]]
    galois_words = orc.fill_uniform(11, list(moduli), n, L * 2 * (L + 1)).reshape(L, 2, L + 1, n)
    word_key = hecuda.EvaluationKey(g, None)
    word_key.setGaloisKey(3, galois_words)
    replaced.setGaloisKey(3, galois_words)
    assert np.array_equal(hecuda.Bfv.applyGalois(g, ct, 3, replaced), hecuda.Bfv.applyGalois(g, ct, 3, word_key))
    single = hecuda.EvaluationKey.fromSerialized(g, **w.python_forms()[rest[0]])  # the element left in place
    assert np.array_equal(hecuda.Bfv.applyGalois(g, ct, 2 * n - 1, replaced), hecuda.Bfv.applyGalois(g, ct, 2 * n - 1, single))
    single.close()
    replaced.close()
    word_key.close()
    # forContext copies a batch-loaded key, and the copy outlives the original
    other = hecuda.Context(n, moduli, 257)
    original = keys[rest[1]]
    relin_want = hecuda.Bfv.relinearize(g, ct3, original)
    copy = original.forContext(other)
    original._copies = {}  # keep the copy alive past the original
    original.close()
    assert np.array_equal(hecuda.Bfv.applyGalois(other, ct, 3, copy), want[rest[1]])
    assert np.array_equal(hecuda.Bfv.relinearize(other, ct3, copy), relin_want)
    copy.close()
    for j in rest[2:]:
        keys[j].close()
    other.close()
    g.close()


def test_load_and_destroy_returns_device_memory():
    import torch

    n = 4096
    g, _ = contexts(n, [27, 28, 28], 17)
    count = 4 * GROUP
    elements = [3, 5, 7, 9, 2 * n - 1]
    w = Wire(n, g.coefficientModuli, 17, True, elements, count, seed=13)
    key_bytes = (1 + len(elements)) * g.L * 2 * (g.L + 1) * n * 8
    staging = 2 * GROUP * w.cts * w.B
    footprint = count * key_bytes + staging + count * w.cts * 4096  # keys, group staging, DRBG chains
    rc, handles = w.many(g)  # warm up the pooled staging and the runtime
    assert rc == 0
    destroy(handles)
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    for _ in range(8):
        rc, handles = w.many(g)
        assert rc == 0, lib().hecuda_last_error()
        destroy(handles)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    assert free0 - free1 <= footprint, (free0 - free1, footprint)
    g.close()


# ---------------------------------------------------------------- 5. errors
def test_errors():
    n = 16
    g, _ = contexts(n, TEST_MODULI_BITS, 1153)
    w = Wire(n, g.coefficientModuli, 1153, True, [3], 3, seed=2)
    launches = hecuda.kernel_launch_count()
    L = lib()

    def call(count=3, relin=1, elements=(3,), element_count=None, poly0=None, seeds=None, ctx=g):
        el = np.ascontiguousarray(elements, dtype=np.uint32)
        poly0 = [p.ctypes.data for p in w.poly0] if poly0 is None else poly0
        seeds = [s.ctypes.data for s in w.seeds] if seeds is None else seeds
        k = max(count, 1)
        out = (C.c_void_p * k)(*([1] * k))
        rc = L.hecuda_evk_create_serialized_many(ctx._h, count, relin, el.ctypes.data if len(el) else None,
                                                 len(el) if element_count is None else element_count,
                                                 (C.c_void_p * 3)(*poly0), (C.c_void_p * 3)(*seeds), out)
        return rc, list(out)

    for j in range(3):  # a null client buffer names the client
        for which in ("poly0", "seeds"):
            ptrs = [p.ctypes.data for p in (w.poly0 if which == "poly0" else w.seeds)]
            ptrs[j] = None
            rc, out = call(**{which: ptrs})
            assert rc == ERR_INVALID_ARGUMENT and not any(out), (j, which)
            assert f"client {j}" in L.hecuda_last_error().decode()
    for kwargs in [dict(elements=(4,)), dict(elements=(1,)), dict(elements=(2 * n + 1,)), dict(elements=(3, 3)),
                   dict(element_count=-1)]:
        rc, out = call(**kwargs)
        assert rc == ERR_INVALID_ARGUMENT and not any(out), kwargs
    for count in (0, -1):
        rc, out = call(count=count)
        assert rc == ERR_INVALID_ARGUMENT, count
    single = hecuda.Context(n, orc.generate_primes([55], False, n), 1153)
    rc, out = call(ctx=single)
    assert rc == ERR_UNSUPPORTED and not any(out)
    single.close()
    assert hecuda.kernel_launch_count() == launches
    # Python: mismatched configs and wrong buffer sizes are refused before the library is called
    forms = w.python_forms()
    for bad, text in [
        (dict(forms[1], relinPoly0=None, relinSeeds=None), "client 1"),
        (dict(forms[1], galois={5: forms[1]["galois"][3]}), "client 1"),
        (dict(forms[1], galois={}), "client 1"),
        (dict(forms[1], relinPoly0=forms[1]["relinPoly0"][:, :-1]), "serializedBufferSizeMismatch"),
        (dict(forms[1], galois={3: (forms[1]["galois"][3][0], forms[1]["galois"][3][1][:1])}), "serializedBufferSizeMismatch"),
    ]:
        with pytest.raises(hecuda.HeError) as err:
            hecuda.EvaluationKey.fromSerializedMany(g, [forms[0], bad, forms[2]])
        assert text in str(err.value), text
    assert hecuda.kernel_launch_count() == launches
    g.close()


# ---------------------------------------------------------------- 6. concurrency
def test_concurrent_batch_loads_are_identical():
    n = 4096
    g, _ = contexts(n, [27, 28, 28], 17)
    w = Wire(n, g.coefficientModuli, 17, True, [3, 5, 2 * n - 1], GROUP + 3, seed=21)
    want = []
    for j in range(len(w.poly0)):
        h = w.single(g, j)
        want.append(w.buffers(h))
        destroy([h])
    errors, results = [], []

    def worker():
        try:
            for _ in range(3):
                rc, handles = w.many(g)
                assert rc == 0, lib().hecuda_last_error()
                results.append([w.buffers(h) for h in handles])
                destroy(handles)
        except Exception as exc:  # noqa: BLE001
            errors.append(exc)

    threads = [threading.Thread(target=worker) for _ in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    assert len(results) == 12
    for got in results:
        for j, (a, b) in enumerate(zip(got, want)):
            for x, y in zip(a, b):
                assert np.array_equal(x, y), j
    g.close()
