"""Processed PIR databases in the reference's file format, on the CPU.

- A known-answer test pins the restatement of ProcessedDatabase.serialize / init(from:context:) (tests/pir_database_io_ref.py)
  with bytes written out by hand.
- tests/emu/database_io_emulate.cu replays the device pipelines on the CPU with the library's own host planning
  (database_io.hpp: tag walk, tag offsets, chunk planner) and the functions its load and serialize kernels call
  (tagged_rows_offset, codec_unpack, codec_pack), chunk by chunk at budgets of a few plaintexts, and must reproduce the
  restatement: the same bytes on save, the same residues and presence flags on load, and the same refusals."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import pir_database_io_ref as ref
from oracle import pir_oracle as opir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_SRC = os.path.join(ROOT, "tests", "emu", "database_io_emulate.cu")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"

KAT_MODULI = [17, 97, 193]  # 5, 7 and 8 bits per coefficient
KAT_P = [[1, 2, 3, 4, 5, 6, 7, 16], [0, 1, 2, 3, 96, 50, 64, 5], [192, 0, 1, 128, 64, 32, 2, 100]]
KAT_P2 = [[16, 15, 0, 0, 0, 0, 0, 1], [96] * 8, [1] * 8]
# [nil, p, nil, p']: version 1, count 4 (LE), then tags and rows.  Row 0 of p at 5 bits: 00001 00010 00011 00100 00101
# 00110 00111 10000 = 08 86 42 98 f0; row 1 at 7 bits, row 2 at 8 bits.
KAT_BYTES = bytes.fromhex(
    "01" "04000000"
    "00"
    "01" "08864298f0" "0004103c0ca005" "c000018040200264"
    "00"
    "01" "83c0000001" "c183060c183060" "0101010101010101")


def test_known_answer():
    plaintexts = [None, np.array(KAT_P, dtype=np.uint64), None, np.array(KAT_P2, dtype=np.uint64)]
    assert ref.serialize_processed_database(8, KAT_MODULI, plaintexts) == KAT_BYTES
    for tail in (b"", b"\x07" * 9):  # trailing bytes are ignored
        loaded = ref.load_processed_database(8, KAT_MODULI, KAT_BYTES + tail)
        assert [p is None for p in loaded] == [True, False, True, False]
        assert np.array_equal(loaded[1], KAT_P) and np.array_equal(loaded[3], KAT_P2)


def test_known_answer_refusals():
    with pytest.raises(ref.DatabaseSerializationError, match="emptyDatabase"):
        ref.serialize_processed_database(8, KAT_MODULI, [None, None])
    with pytest.raises(ref.DatabaseSerializationError, match=r"Version\(serializationVersion: 2, expected: 1\)"):
        ref.load_processed_database(8, KAT_MODULI, b"\x02" + KAT_BYTES[1:])
    with pytest.raises(ref.DatabaseSerializationError, match=r"PlaintextTag\(tag: 2\)"):
        ref.load_processed_database(8, KAT_MODULI, KAT_BYTES[:5] + b"\x02" + KAT_BYTES[6:])
    for end in (0, 3, 5, 7, 26, 47):
        with pytest.raises(ref.DatabaseSerializationError, match="corruptedData"):
            ref.load_processed_database(8, KAT_MODULI, KAT_BYTES[:end])


# ---- the device pipelines' host replay -------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    binary = str(tmp_path_factory.mktemp("emu") / "database_io_emulate")
    subprocess.check_call([NVCC, "-O1", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", binary, EMU_SRC])
    return binary


def run(binary, mode, n, moduli, budget, text):
    args = [binary, mode, str(n), str(budget), str(len(moduli))] + [str(q) for q in moduli]
    return subprocess.run(args, input=text, capture_output=True, text=True, check=True).stdout.splitlines()


def parse_plan(lines):
    tags = [int(v) for v in lines[0].split()[1:]]
    chunks = []
    for line in lines[1:]:
        if not line.startswith("chunk "):
            break
        chunks.append(tuple(int(v) for v in line.split()[1:]))
    return tags, chunks, lines[1 + len(chunks):]


def check_plan(tags, chunks, count, budget):
    """Whole plaintexts, consecutive, covering every one; a chunk exceeds the budget only as a single plaintext."""
    assert [c[0] for c in chunks] == list(np.cumsum([0] + [c[1] for c in chunks[:-1]]))
    assert sum(c[1] for c in chunks) == count
    for first, n in chunks:
        size = tags[first + n] - tags[first]
        assert n >= 1 and (size <= budget or n == 1)
        if first + n < count:  # greedy: the next plaintext would not have fit
            assert tags[first + n + 1] - tags[first] > budget


def emulate_load(binary, n, moduli, budget, data):
    lines = run(binary, "load", n, moduli, budget, (data.hex() or ".") + "\n")
    walk = [int(v) for v in lines[0].split()[1:]]
    if walk[0] or not walk[3]:
        return walk, None
    tags, chunks, rest = parse_plan(lines[1:])
    table = np.array([[int(v) for v in line.split()] for line in rest[:-1]], dtype=np.uint64).reshape(walk[3], -1)
    return walk, (tags, chunks, table[:, 0], table[:, 1:].reshape(walk[3], len(moduli), n), int(rest[-1].split()[1]))


def emulate_save(binary, n, moduli, budget, plaintexts):
    text = f"{len(plaintexts)}\n" + "".join(
        ("0 " + " ".join(["0"] * (n * len(moduli))) if p is None else "1 " + " ".join(str(int(v)) for v in np.ravel(p))) + "\n"
        for p in plaintexts)
    lines = run(binary, "save", n, moduli, budget, text)
    tags, chunks, rest = parse_plan(lines)
    return tags, chunks, bytes.fromhex(rest[0]), bytes.fromhex(rest[1])


def moduli_of(bits, n):
    from oracle import oracle as orc
    return orc.generate_primes(bits, False, n)[: len(bits)]


# (N, moduli or bit sizes, plaintext count, nil pattern period)
SHAPES = [
    (8, KAT_MODULI, 9, 3),
    (16, [27, 28, 28], 13, 4),
    (64, [27, 28, 28], 11, 5),        # rows of 216 / 224 bytes: the 8-byte kernel path
    (64, [55, 55, 55, 55], 7, 2),
    (256, [61, 60, 62], 6, 7),
]


def random_plaintexts(rng, n, moduli, count, period):
    out = []
    for i in range(count):
        if i % period == 1:
            out.append(None)
            continue
        rows = np.stack([np.array([int(v) for v in rng.integers(0, q, size=n, dtype=np.uint64)], dtype=np.uint64)
                         for q in moduli])
        rows[:, 0] = [q - 1 for q in moduli]  # the largest residue of every row
        out.append(rows)
    return out


@pytest.mark.parametrize("n,mods,count,period", SHAPES)
def test_pipelines_replay_the_format(emu, n, mods, count, period):
    moduli = mods if n == 8 else moduli_of(mods, n)
    rng = np.random.default_rng(n * 31 + count)
    plaintexts = random_plaintexts(rng, n, moduli, count, period)
    expected = ref.serialize_processed_database(n, moduli, plaintexts)
    size = opir.serialization_byte_count(n, moduli)
    words = all((n * opir.ceil_log2(q)) % 64 == 0 for q in moduli)
    tags_expected = list(np.cumsum([5] + [1 + (size if p is not None else 0) for p in plaintexts]))
    exact = tags_expected[3] - tags_expected[0]  # the first chunk ends exactly on the budget
    # budgets: below one plaintext, exactly three plaintexts, a few, and everything
    for budget in (size // 2, exact, 2 * size + 7, len(expected)):
        tags, chunks, by_bytes, by_words = emulate_save(emu, n, moduli, budget, plaintexts)
        assert tags == tags_expected
        check_plan(tags, chunks, count, budget)
        assert by_bytes == expected
        if words:
            assert by_words == expected
        if budget == exact:
            assert chunks[0] == (0, 3)
        walk, loaded = emulate_load(emu, n, moduli, budget, expected + b"\x05\x06")
        assert walk[0] == 0 and walk[3] == count
        ltags, lchunks, present, rows, bad = loaded
        assert ltags == tags and lchunks == chunks and bad == -1
        assert list(present) == [p is not None for p in plaintexts]
        for p, got in zip(plaintexts, rows):
            assert np.array_equal(got, p if p is not None else np.zeros_like(got))
        assert len(chunks) > 1 or budget >= len(expected) - 5


def test_load_flags_the_first_residue_not_below_its_modulus(emu):
    n, moduli = 16, moduli_of([27, 28, 28], 16)
    plaintexts = random_plaintexts(np.random.default_rng(3), n, moduli, 8, 4)
    for index, row in ((6, 2), (3, 0)):  # the second one comes first in stream order
        plaintexts[index][row, 5] = moduli[row]  # one past the largest residue (fits the row's bit width)
    data = ref.serialize_processed_database(n, moduli, plaintexts)
    assert ref.load_processed_database(n, moduli, data)[3][0, 5] == moduli[0]  # the reference accepts it
    size = opir.serialization_byte_count(n, moduli)
    for budget in (size, 3 * size, len(data)):
        walk, loaded = emulate_load(emu, n, moduli, budget, data)
        assert walk[0] == 0 and loaded[4] == 3 * len(moduli) + 0


def test_tag_walk_refuses_what_the_reference_refuses(emu):
    n, moduli = 8, KAT_MODULI
    data = KAT_BYTES
    cases = {
        b"": (3, -1),                                     # truncated header
        b"\x02" + data[1:]: (1, -1),                      # version
        data[:3]: (3, -1),
        data[:5] + b"\x02" + data[6:]: (2, 0),            # tag of plaintext 0
        data[:27] + b"\x09" + data[28:]: (2, 2),          # tag of plaintext 2
        data[:27]: (3, 2),                                # the buffer ends before plaintext 2's tag
        data[:40]: (3, 3),                                # inside plaintext 3's rows
        data[:1] + (1000).to_bytes(4, "little") + data[5:]: (3, -1),  # a count that cannot fit the buffer
    }
    for raw, (error, at) in cases.items():
        walk, _ = emulate_load(emu, n, moduli, 64, raw)
        assert (walk[0], walk[2]) == (error, at), raw.hex()
        with pytest.raises(ref.DatabaseSerializationError):
            ref.load_processed_database(n, moduli, raw)
    walk, _ = emulate_load(emu, n, moduli, 64, b"\x07" + data[1:])
    assert walk[1] == 7
    walk, loaded = emulate_load(emu, n, moduli, 64, b"\x01\x00\x00\x00\x00")
    assert walk == [0, 0, -1, 0]
