"""CPU-side verification of the keyword-PIR device code (csrc/sha256.cuh, csrc/keyword_pir.cuh) and the placement
(csrc/cuckoo.hpp).

tests/emu/keyword_pir_emulate.cu evaluates the very same __host__ __device__ functions the hash, candidate-index and
bucket-serialization kernels call, and the host placement that hecuda_cuckoo_table_create runs:
  - SHA-256 equals hashlib for every message length 0..300 (the padding boundaries 55, 56, 63, 64, 119, 120 included);
  - the serialized buckets equal the oracle's (oracle/keyword_oracle.py) byte for byte, for both generators."""
import hashlib
import os
import random
import shutil
import subprocess

import pytest

from oracle import keyword_oracle as K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_SRC = os.path.join(ROOT, "tests", "emu", "keyword_pir_emulate.cu")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    binary = str(tmp_path_factory.mktemp("emu") / "keyword_pir_emulate")
    subprocess.check_call([NVCC, "-O1", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", binary, EMU_SRC])
    return binary


def run(binary, args, text):
    return subprocess.run([binary] + [str(a) for a in args], input=text, capture_output=True, text=True,
                          check=True).stdout.splitlines()


def test_sha256_matches_hashlib(emu):
    rng = random.Random(5)
    messages = [bytes(rng.randrange(256) for _ in range(n)) for n in range(301)]
    lines = run(emu, ["sha"], "".join((m.hex() or ".") + "\n" for m in messages))
    assert len(lines) == len(messages)
    for m, line in zip(messages, lines):
        digest, first8 = line.split()
        assert digest == hashlib.sha256(m).hexdigest(), len(m)
        assert int(first8) == K.keyword_hash(m)


def emulate_table(binary, config, rows, rng_kind, seed):
    fixed = config.bucket_count or 0
    args = ["table", config.hash_function_count, config.max_eviction_count, config.max_serialized_bucket_size,
            config.slot_count, int(config.multiple_tables), fixed, config.expansion_factor, config.target_load_factor,
            rng_kind, seed]
    lines = run(binary, args, "".join(f"{k.hex() or '.'} {v.hex() or '.'}\n" for k, v in rows))
    if lines and lines[0].startswith("error"):
        return lines[0]
    return [bytes.fromhex(line) for line in lines]


def mixed_rows(seed, count, sizes=(0, 1, 2, 30, 60)):
    r = random.Random(seed)
    return [(bytes(r.randrange(256) for _ in range(12)), bytes(r.randrange(256) for _ in range(r.choice(sizes))))
            for _ in range(count)]


def summarize_rows():
    rng = K.TestRng(1)
    rows = K.random_keyword_pir_database(100, 10, rng)
    return rows, rng.counter


CASES = {
    "summarize": lambda: (K.CuckooTableConfig(2, 100, 50), *summarize_rows()),
    "evictions20": lambda: (K.CuckooTableConfig(2, 20, 50), K.random_keyword_pir_database(300, 10, K.TestRng(0)), 0),
    "slots7": lambda: (K.CuckooTableConfig(2, 100, 5000, slot_count=7), K.random_keyword_pir_database(300, 10, K.TestRng(3)), 0),
    "h3": lambda: (K.CuckooTableConfig(3, 100, 100), K.random_keyword_pir_database(200, 20, K.TestRng(7)), 4),
    "single_table": lambda: (K.CuckooTableConfig(2, 100, 80, multiple_tables=False),
                             K.random_keyword_pir_database(150, 10, K.TestRng(9)), 1),
    "fixed": lambda: (K.CuckooTableConfig(2, 100, 50, bucket_count=100), K.random_keyword_pir_database(100, 10, K.TestRng(0)), 0),
    "mixed_divergent": lambda: (K.CuckooTableConfig(2, 100, 100), mixed_rows(3, 100), 10),
    "mixed_zero_length": lambda: (K.CuckooTableConfig(2, 100, 120), mixed_rows(11, 200, (0, 0, 5, 40)), 2),
    "duplicates": lambda: (K.CuckooTableConfig(2, 100, 50), [(b"a", b"1"), (b"b", b"2"), (b"a", b"3"), (b"", b"")] * 3, 0),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("rng_kind", [0, 1])
def test_buckets_match_the_oracle(emu, case, rng_kind):
    config, rows, seed = CASES[case]()
    oracle_rng = K.TestRng(seed) if rng_kind == 0 else K.SplitMix64(seed)
    expected = K.CuckooTable(config, rows, oracle_rng).serialize_buckets()
    assert emulate_table(emu, config, rows, rng_kind, seed) == expected


def test_errors_match_the_oracle(emu):
    rows = K.random_keyword_pir_database(100, 10, K.TestRng(0))
    assert emulate_table(emu, K.CuckooTableConfig(2, 100, 50, bucket_count=10), rows, 0, 0).startswith(
        "error failedToConstructCuckooTable")
    assert emulate_table(emu, K.CuckooTableConfig(2, 100, 30), [(b"k", bytes(40))], 0, 0).startswith(
        "error failedToConstructCuckooTable")
