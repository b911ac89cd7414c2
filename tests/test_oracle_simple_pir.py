"""CPU checks of the SimplePIR oracle (oracle/simple_pir_oracle.py): the adjoint identity the device hint uses against
the materialised DB' . A, Swift's rounding in computingParams, and a noiseless selection query decoding every entry."""
import random

import numpy as np
import pytest

from oracle import simple_pir_oracle as osp


@pytest.mark.parametrize("n,columns", [(8, 21), (16, 40), (32, 64)])
def test_adjoint_hint_equals_materialised_product(n, columns):
    rng = np.random.default_rng(n)
    p = osp.ntt_friendly_mod(20, n)
    polys = osp.a_polynomials(bytes(range(32)), n, -(-columns // n), p)
    db = rng.integers(0, 1 << 14, size=(5, columns)).astype(np.uint64)
    dense = osp.mulmod_matrix(db, osp.a_matrix(polys, columns, p), p)
    assert np.array_equal(dense, osp.hint_adjoint(db, polys, p))
    exact = [[sum(int(db[r, k]) * int(v) for k, v in enumerate(col)) % p for col in osp.a_matrix(polys, columns, p).T]
             for r in range(5)]
    assert np.array_equal(dense, np.array(exact, dtype=np.uint64))


def test_swift_rounding_and_truncation():
    assert [osp.swift_rounded(x) for x in (0.5, 1.5, 2.5, 0.49)] == [1, 2, 3, 0]
    assert [round(x) for x in (0.5, 2.5)] == [0, 2]  # what Python's round would have given
    a = osp.computing_params(14, 1 << 20, 256)
    assert (a["chunks_per_entry"], a["database_columns"]) == (1, 1 << 20)
    b = osp.computing_params(14, 4096, 256 * 1024)
    assert (b["chunks_per_entry"], b["database_columns"]) == (6, 24576)
    assert osp.shape(14, 256 * 1024, 1, 6)[2] == 24967
    assert osp.ntt_friendly_mod(42, 2048) == 4398046523393


@pytest.mark.parametrize("pt,ct,count,size", [(7, 28, 600, 20), (14, 42, 600, 20), (7, 28, 20, 600), (14, 42, 20, 600)])
def test_noiseless_selection_decodes_entries(pt, ct, count, size):
    rng = random.Random(pt + count)
    entries = np.array([[rng.randrange(256) for _ in range(size)] for _ in range(count)], dtype=np.uint8)
    prm = osp.computing_params(pt, count, size)
    epc, cpe, k = prm["entries_per_column"], prm["chunks_per_entry"], prm["database_columns"]
    db = osp.process_database(entries, pt, epc, cpe, k)
    for index in rng.sample(range(count), 5):
        resp = osp.response(db, osp.selection_request(index, pt, ct, epc, cpe, k), ct)
        assert osp.decode_noiseless(resp, index, pt, ct, size, epc, cpe) == entries[index].tobytes()


NOISELESS_CASES = [  # SimplePirTests.noiselessSample: (pt, ct, N, entryCount, entrySize) -> (cpe > 1, aPolyCount > 1)
    ((8, 9, 16, 1, 1), (False, False)), ((8, 9, 8, 10, 1), (False, True)), ((4, 8, 8, 1, 1), (True, False)),
    ((4, 8, 8, 10, 62), (True, True))]


@pytest.mark.parametrize("case,expect", NOISELESS_CASES)
def test_noiseless_sample_cases(case, expect):
    pt, ct, n, count, size = case
    prm = osp.computing_params(pt, count, size)
    k, cpe = prm["database_columns"], prm["chunks_per_entry"]
    polys_count = -(-k // n)
    assert (cpe > 1, polys_count > 1) == expect
    p = osp.ntt_friendly_mod(ct, n)
    polys = osp.a_polynomials(bytes(32), n, polys_count, p)
    s = osp.secret_polys(np.random.default_rng(n + count), cpe, n)
    matrix = osp.noiseless_sample(s, osp.a_matrix(polys, k, p), p)
    assert np.array_equal(matrix, osp.noiseless_sample_polynomial(s, polys, k, p))


def test_ternary_secret_key_maps_correctly_after_mod_switch():
    ct, n = 42, 2048
    p = osp.ntt_friendly_mod(ct, n)
    s = osp.secret_polys(np.random.default_rng(0), 1, n)
    switched = osp.mod_switch(s % p, p, ct)
    assert set(int(v) for v in switched.reshape(-1)) == {0, 1, (1 << ct) - 1}


@pytest.mark.parametrize("pt,ct,count,size", [(7, 28, 600, 20), (14, 42, 600, 20), (7, 28, 20, 600), (14, 42, 20, 600)])
def test_encrypted_round_trip(pt, ct, count, size):
    """runEncryptDecryptRoundTripTest at N = 1024 on the oracle alone: process, the client's encrypted queries with
    error, the response, decryption of 5 random entries."""
    rng = np.random.default_rng(pt * count + size)
    entries = rng.integers(0, 256, size=(count, size), dtype=np.uint8)
    prm = osp.computing_params(pt, count, size)
    db = osp.process_database(entries, pt, prm["entries_per_column"], prm["chunks_per_entry"], prm["database_columns"])
    seed = bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    hint = osp.hint(db, seed, 1024, osp.ntt_friendly_mod(ct, 1024))
    prm.update(N=1024, pt=pt, ct=ct, entry_size=size)
    client = osp.Client(prm, hint, seed, rng)
    for index in rng.choice(count, 5, replace=False):
        query, results = client.query(int(index))
        assert client.decrypt(osp.response(db, query, ct), results, int(index)) == entries[index].tobytes()
