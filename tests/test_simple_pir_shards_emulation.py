"""CPU replay of sharded SimplePIR's index maps (csrc/simple_pir.cuh) through tests/emu/simple_pir_shards_emulate.cu.

- The grouped response's plan and item decode: every (shard, row CTA, query-tile pair) is one item per K range, and
  the K ranges partition the shard's column tiles, for ragged shards, S in {1, 5, 32, 33} and client counts whose
  query padding differs per shard; no launch holds more than 32 shards.
- The chunk locations' inversion and the row -> piece map rebuild shardDatabase's shard matrices byte for byte
  (tests/simple_pir_shards_ref.py) for random maps over variable entry sizes, and refuse locations that are not a
  permutation of every shard's rows or leave a shard empty."""
import os
import random
import shutil
import subprocess
from collections import defaultdict

import numpy as np
import pytest

import simple_pir_shards_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_SRC = os.path.join(ROOT, "tests", "emu", "simple_pir_shards_emulate.cu")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
SMS, MAX_SHARDS, MIN_SPLIT = 132, 32, 64  # an H100 SXM's SMs; simple_pir.cu's kMaxShards and kMinSplitTiles


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    binary = str(tmp_path_factory.mktemp("emu") / "simple_pir_shards_emulate")
    subprocess.check_call([NVCC, "-O1", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", binary, EMU_SRC])
    return binary


def plan(binary, shards):
    text = f"{len(shards)}\n" + "".join(f"{m} {tiles} {q}\n" for m, tiles, q in shards)
    out = subprocess.run([binary, "items", str(SMS), str(MAX_SHARDS), str(MIN_SPLIT)], input=text, capture_output=True,
                         text=True, check=True).stdout
    return [tuple(int(v) for v in line.split()) for line in out.splitlines()]


@pytest.mark.parametrize("shard_count", [1, 5, 32, 33])
@pytest.mark.parametrize("clients", [1, 3, 17])
def test_items_cover_every_cta_once_and_partition_k(emu, shard_count, clients):
    rng = random.Random(shard_count * 100 + clients)
    shards = []
    for _ in range(shard_count):
        m = rng.choice([1, 30, 127, 128, 129, 1000])
        k = rng.choice([1, 31, 32, 700, 64 * 32 * 3 + 5, 40000])
        cpe = rng.choice([1, 2, 3, 6])
        shards.append((m, -(-k // 32), clients * 2 * cpe))  # two requests per shard
    items = plan(emu, shards)
    launches = defaultdict(set)
    seen = defaultdict(list)
    for launch, s, row_cta, pair, kb, ke in items:
        launches[launch].add(s)
        seen[(s, row_cta, pair)].append((kb, ke))
    assert all(len(group) <= MAX_SHARDS for group in launches.values())
    assert len(launches) == -(-shard_count // MAX_SHARDS)
    for s, (m, tiles, q) in enumerate(shards):
        for row_cta in range(-(-m // 128)):
            for pair in range(-(-q // 16)):
                ranges = sorted(seen.pop((s, row_cta, pair)))
                assert ranges[0][0] == 0 and ranges[-1][1] == tiles
                assert all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
                assert all(kb < ke for kb, ke in ranges)
    assert not seen  # no item outside the shards' CTAs


def test_one_small_shard_splits_k_like_the_single_database_call(emu):
    """A lone shard of one row CTA and one query pair over 3 x 64 + 5 tiles: K splits into 3 ranges of >= 64 tiles."""
    items = plan(emu, [(100, 64 * 3 + 5, 1)])
    assert [(kb, ke) for *_, kb, ke in items] == [(0, 66), (66, 132), (132, 197)]


def rows(binary, sizes, values, shard_count, chunk_size, locations):
    text = f"{len(sizes)} {shard_count} {chunk_size}\n{' '.join(map(str, sizes))}\n{' '.join(map(str, values))}\n" \
           f"{' '.join(str(int(v)) for v in np.asarray(locations).reshape(-1))}\n"
    out = subprocess.run([binary, "rows"], input=text, capture_output=True, text=True, check=True).stdout.split("\n")
    if out[0] == "refused":
        return None
    got = [[] for _ in range(shard_count)]
    for line in out[1:]:
        if line:
            s, hexrow = line.split()
            got[int(s)].append(bytes.fromhex(hexrow))
    return [np.frombuffer(b"".join(r), dtype=np.uint8).reshape(len(r), chunk_size) for r in got]


@pytest.mark.parametrize("seed", range(4))
def test_row_pieces_rebuild_the_shards(emu, seed):
    rng = np.random.default_rng(seed)
    shard_count, chunk_size = int(rng.integers(1, 7)), int(rng.integers(1, 40))
    entries = [(i, rng.integers(0, 256, size=int(rng.integers(0, 150)), dtype=np.uint8).tobytes()) for i in range(60)]
    perms = [rng.permutation(shard_count) for _ in entries]
    mapped, shards = ref.shard_database(entries, shard_count, chunk_size, perms)
    locations = [loc for _, _, chunks in mapped for loc in chunks]
    values = [b for _, v in entries for b in v]
    got = rows(emu, [len(v) for _, v in entries], values, shard_count, chunk_size, locations)
    if any(len(s) == 0 for s in shards):
        assert got is None  # an empty shard is refused
        return
    assert len(got) == shard_count
    for a, b in zip(got, shards):
        assert np.array_equal(a, b)


def test_locations_that_are_not_a_permutation_are_refused(emu):
    sizes, values = [10, 10, 10, 10], list(range(40))
    good = [(0, 0), (1, 0), (0, 1), (1, 1)]  # chunk size 10: one chunk per entry
    assert rows(emu, sizes, values, 2, 10, good) is not None
    for bad in ([(0, 0), (1, 0), (0, 0), (1, 1)],  # a row twice
                [(0, 0), (1, 0), (0, 2), (1, 1)],  # past the shard's rows
                [(0, 0), (2, 0), (0, 1), (1, 1)],  # no such shard
                [(0, 0), (0, 1), (0, 2), (0, 3)]):  # shard 1 empty
        assert rows(emu, sizes, values, 2, 10, bad) is None
