"""SimplePIR's two slab loops past their first slab.  The server's hint (compute_hint, csrc/simple_pir.cu) and the
client's query precompute (precompute_device, csrc/simple_pir_client.cu) each work through their rows in slabs of at
most 2^25 words, so every slab after the first reads and writes at a row offset r0 > 0.  Every shape here reaches at
least three slabs with a partial last one:

  * the hint at N 16 with 4096 A-polynomials (512-row slabs) and 1025 DB' rows, at the widest hint moduli (ct 61
    UInt64, ct 31 UInt32), whose lazy Eval inner product must reduce inside its 4096-term sum: chosen rows, including
    both sides of each boundary, bit-exact against oracle/simple_pir_oracle.py;
  * the client's precompute at the same N and K with chunksPerEntry 3 and 400 queries (1200 secret rows in slabs of
    512, 512 and 176), so the chunks of queries 170 and 341 lie on both sides of a boundary.  Those two, the first and
    last query and the first query wholly inside each later slab are bit-exact against tests/simple_pir_client_ref.py;
    every query decrypts back to its entry through the device server; the device-pointer precompute equals the host
    call.
"""
import ctypes as C
import os
import re
from dataclasses import dataclass

import numpy as np
import pytest

import hecuda
import simple_pir_client_ref as ref
from hecuda import simple_pir as sp
from oracle import simple_pir_oracle as osp

pytestmark = pytest.mark.gpu

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "swift-homomorphic-encryption_b200",
                    "csrc")


def slab_words(source: str, name: str) -> int:
    """A slab constant `constexpr int64_t name = a ll << b;` as the library is built with it."""
    with open(os.path.join(CSRC, source)) as f:
        m = re.search(rf"constexpr int64_t {name} = (\d+)ll << (\d+);", f.read())
    assert m, f"{name} not found in {source}"
    return int(m.group(1)) << int(m.group(2))


HINT_SLAB_WORDS = slab_words("simple_pir.cu", "kHintSlabWords")
CLIENT_SLAB_WORDS = slab_words("simple_pir_client.cu", "kSlabWords")


def slab_plan(rows: int, blocks: int, n: int, words: int):
    """Both loops' slab: max(1, min(rows, words / (blocks N))) rows -> (slab rows, slab count)."""
    slab = max(1, min(rows, words // (blocks * n)))
    return slab, -(-rows // slab)


def enc(pt, ct, n, std=3.2):
    return sp.SimplePirEncryptionParams(pt, ct, n, std, "unchecked")


def process(entries: np.ndarray, prm: sp.SimplePirParameters, scalar):
    """hecuda_simple_pir_process at the given parameters (SimplePirServer.process would choose its own)."""
    lib = hecuda.load_library()
    hint = np.zeros((prm.columnSize, prm.latticeDimension), dtype=scalar)
    seed = np.frombuffer(prm.seed, dtype=np.uint8).copy()
    h = C.c_void_p()
    cp = prm._c(np.dtype(scalar).itemsize * 8)
    assert lib.hecuda_simple_pir_process(entries.ctypes.data, entries.shape[0], C.byref(cp), seed.ctypes.data,
                                         hint.ctypes.data, C.byref(h)) == 0
    return sp.SimplePirDatabase(h, prm, scalar), hint


N, K = 16, 65536  # 4096 A-polynomials: 512 rows per slab in both loops


@pytest.mark.parametrize("ct,scalar", [(61, np.uint64), (31, np.uint32)], ids=["uint64-ct61", "uint32-ct31"])
def test_hint_past_the_first_slab_at_the_widest_modulus(ct, scalar):
    m = 1025  # pt 8: one DB' row per entry byte
    slab, slabs = slab_plan(m, K // N, N, HINT_SLAB_WORDS)
    assert slabs >= 3 and m % slab, (slab, slabs)  # 512, 512, 1
    rng = np.random.default_rng(ct)
    prm = sp.SimplePirParameters(enc(8, ct, N), m, 1, 1, K, rng.integers(0, 256, 32, dtype=np.uint8).tobytes())
    assert prm.columnSize == m and prm.aPolyCount == K // N
    entries = rng.integers(0, 256, size=(K, m), dtype=np.uint8)
    # pt 8, one entry per column and one chunk per entry: DB' is the transposed byte matrix
    assert np.array_equal(osp.process_database(entries[:40], 8, 1, 1, 40), entries[:40].T)
    database, hint = process(entries, prm, scalar)
    assert np.array_equal(database.export(), entries.T)
    rows = sorted({0, slab - 1, slab, slab + 1, 2 * slab - 1, 2 * slab, m - 1} |
                  {int(r) for r in rng.choice(m, 6, replace=False)})
    p = osp.ntt_friendly_mod(ct, N)
    assert p.bit_length() == ct + 1
    expect = osp.hint(entries.T[rows], prm.seed, N, p)  # each hint row depends only on its own DB' row
    wrong = [(r, r // slab) for i, r in enumerate(rows) if not np.array_equal(hint[r].astype(np.uint64), expect[i])]
    assert not wrong, f"(hint row, slab) {wrong}"
    database.close()


# The client: chunksPerEntry 3, one entry per column, 400 queries -> 1200 secret rows.  pt 8 and 30-byte entries give
# 10 hint rows.  UInt32 runs at ct 30: there the reference's double-width results sum cannot wrap at N 16, so every
# query must decrypt.
CPE, COUNT, SIZE = 3, 400, 30


@dataclass
class Batch:
    scalar: type
    prm: sp.SimplePirParameters
    entries: np.ndarray
    server: sp.SimplePirServer
    client: sp.SimplePirClient
    secret_seeds: list
    error_seeds: list
    indices: np.ndarray
    queries: np.ndarray
    results: np.ndarray
    checked: list  # the queries compared with the Python reference


def client_plan():
    """The client's slabs at COUNT queries; the queries whose chunks straddle a boundary, and the ones checked."""
    rows = COUNT * CPE
    slab, slabs = slab_plan(rows, K // N, N, CLIENT_SLAB_WORDS)
    assert slabs >= 3 and rows % slab, (slab, slabs)  # 512, 512, 176
    assert slab % CPE, slab
    straddling = [q for q in range(COUNT) if q * CPE // slab != (q * CPE + CPE - 1) // slab]
    assert len(straddling) == slabs - 1, straddling  # every boundary splits a query: 170 (rows 510-512), 341
    firsts = [-(-b * slab // CPE) for b in range(1, slabs)]  # the first query wholly inside each later slab
    return straddling, sorted({0, COUNT - 1, *straddling, *firsts})


@pytest.fixture(scope="module", params=[(30, np.uint32), (61, np.uint64)], ids=["uint32-ct30", "uint64-ct61"])
def batch(request):
    ct, scalar = request.param
    rng = np.random.default_rng(ct + 1)
    seed = rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
    prm = sp.SimplePirParameters(enc(8, ct, N), SIZE, 1, CPE, K, seed)
    entries = rng.integers(0, 256, size=(K // CPE, SIZE), dtype=np.uint8)  # the last of the K columns stays empty
    database, hint = process(entries, prm, scalar)
    server = sp.SimplePirServer(database, hint, prm, scalar)
    client = sp.SimplePirClient(sp.DefaultQueryGenerator(prm, hint, scalar))
    ss = [rng.integers(0, 256, 32, dtype=np.uint8).tobytes() for _ in range(COUNT)]
    es = [rng.integers(0, 256, 32, dtype=np.uint8).tobytes() for _ in range(COUNT)]
    indices = rng.integers(0, len(entries), size=COUNT)
    indices[-1] = len(entries) - 1  # its last chunk's delta lands in column K - 2
    q, r = client.queryGenerator.precompute(COUNT, indices, ss, es)
    _, checked = client_plan()
    yield Batch(scalar, prm, entries, server, client, ss, es, indices, q, r, checked)
    client.queryGenerator.close()
    database.close()


def test_precompute_past_the_first_slab(batch):
    prm = batch.prm
    ct, bits = prm.ciphertextModulusBits, np.dtype(batch.scalar).itemsize * 8
    d = dict(N=N, pt=8, ct=ct, entries_per_column=1, chunks_per_entry=CPE, database_columns=K)
    wrong = []
    for i in batch.checked:  # about a second of Python AES and integer arithmetic each
        eq, er, _ = ref.precompute(d, batch.server.hint, prm.seed, batch.secret_seeds[i], batch.error_seeds[i],
                                   int(batch.indices[i]), bits, 3.2)
        if not np.array_equal(batch.queries[i].astype(np.uint64), eq):
            wrong.append((i, "queries"))
        if not np.array_equal(batch.results[i].astype(np.uint64), er):
            wrong.append((i, "resultsWithoutResponse"))
    assert not wrong, wrong


def test_every_query_decrypts_its_entry(batch):
    """Device response and device decryption: each of the 400 queries, in every slab and across both boundaries,
    must return its entry's bytes."""
    responses = batch.server.computeResponses(batch.queries)
    got = batch.client.decryptMany(responses, batch.results, batch.indices)
    wrong = [i for i in range(COUNT) if got[i].tobytes() != batch.entries[batch.indices[i]].tobytes()]
    assert not wrong, f"queries not decrypted to their entries: {wrong} (straddling {client_plan()[0]})"


def test_device_precompute_matches_the_host_call(batch):
    """precomputeDevice on the caller's stream, then the device-pointer response and decryption in stream order."""
    torch = pytest.importorskip("torch")
    prm = batch.prm
    tdt = torch.int64 if batch.scalar == np.uint64 else torch.int32
    d_ss = torch.from_numpy(np.frombuffer(b"".join(batch.secret_seeds), dtype=np.uint8).copy()).cuda()
    d_es = torch.from_numpy(np.frombuffer(b"".join(batch.error_seeds), dtype=np.uint8).copy()).cuda()
    d_idx = torch.from_numpy(batch.indices.astype(np.int64)).cuda()
    d_q = torch.zeros((COUNT, CPE, K), dtype=tdt, device="cuda")
    d_r = torch.zeros((COUNT, CPE, prm.columnSize), dtype=tdt, device="cuda")
    d_resp = torch.zeros_like(d_r)
    d_out = torch.zeros((COUNT, SIZE), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())  # the buffers' fills run first
    with torch.cuda.stream(s):
        batch.client.precomputeDevice(d_ss.data_ptr(), d_es.data_ptr(), d_idx.data_ptr(), COUNT, d_q.data_ptr(),
                                      d_r.data_ptr(), s.cuda_stream)
        batch.server.computeResponsesDevice(d_q.data_ptr(), COUNT, d_resp.data_ptr(), s.cuda_stream)
        batch.client.decryptDevice(d_resp.data_ptr(), d_r.data_ptr(), d_idx.data_ptr(), COUNT, d_out.data_ptr(),
                                   s.cuda_stream)
    s.synchronize()
    assert np.array_equal(d_q.cpu().numpy().view(batch.scalar), batch.queries)
    assert np.array_equal(d_r.cpu().numpy().view(batch.scalar), batch.results)
    assert np.array_equal(d_out.cpu().numpy(), batch.entries[batch.indices])
