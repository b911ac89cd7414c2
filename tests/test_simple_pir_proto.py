"""CPU checks of SimplePIR's protobuf messages:

- tests/simple_pir_proto_ref.py is pinned by hand-written known-answer byte strings and cross-checked against
  google.protobuf with descriptors built from the field tables of pir/v1/simple_pir.proto and api/pir/v1/pir.proto:
  packed, split-packed and unpacked data, and the values 0, 127, 128, 2^28, 2^32 - 1, 2^32, 2^ct - 1 and 2^64 - 1;
- the library's host-only calls (hecuda_simple_pir_request_write / _fields_read / _response_read and the
  SimplePIRConfig calls) reproduce the restatement, refusals included;
- tests/emu/simple_pir_proto_emulate.cu runs the library's request walk and the device decode and encode maps
  (simple_pir.cuh) on the CPU: every decoded value lands where split_shards_kernel puts its digits, every refusal is
  flagged, and the encoded responses are the restatement's bytes."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import hecuda
import simple_pir_proto_ref as ref
from hecuda import simple_pir as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_SRC = os.path.join(ROOT, "tests", "emu", "simple_pir_proto_emulate.cu")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CT = 42
VALUES = [0, 127, 128, 1 << 28, (1 << 32) - 1, 1 << 32, (1 << CT) - 1, (1 << 64) - 1]
SEED = bytes(range(32))


# ---- known answers (written out by hand from the .proto field numbers and the varint rules)

def test_known_answers():
    # SimplePIRRequest { request { row_count 1, col_count 2, data [1, 300] }, shard_index 3, configuration_hash "h" }
    assert ref.encode_request(1, 2, [1, 300], 3, b"h") == bytes.fromhex("0a09 0801 1002 1a03 01ac02 1003 1a0168")
    # a zero shard index and an empty hash are omitted; an empty request matrix is still written
    assert ref.encode_request(0, 0, []) == bytes.fromhex("0a00")
    # SimplePIRResponse { response { col_count 5 } }: a 0 x 5 reply
    assert ref.encode_response(0, 5, []) == bytes.fromhex("0a02 1005")
    # 2^64 - 1 takes ten bytes
    assert ref.encode_response(1, 1, [(1 << 64) - 1]) == bytes.fromhex("0a10 0801 1001 1a0a ffffffffffffffffff01")
    # SimplePIREncryptionParams { 2048, 6.4 (fixed64), 14, 42 }
    assert ref.encode_encryption_params(2048, 6.4, 14, 42) == bytes.fromhex("0880 10 119a9999999999 1940 180e 202a")
    # DatabaseMapping { entries { original_index 7, size 3, chunks { shard 0, index 0 }, chunks { 1, 2 } }, chunk_size 2 }
    assert ref.encode_database_mapping([(7, 3, [(0, 0), (1, 2)])], 2) == bytes.fromhex(
        "0a0c 0807 1003 1a00 1a04 08011002 1002")


def test_capacity_bounds_every_response():
    rng = np.random.default_rng(1)
    for ct in (28, 32, 42, 61):
        for rows, cols in ((0, 5), (1, 1), (3, 200), (17, 30)):
            data = [(1 << ct) - 1] * (rows * cols)
            assert len(ref.encode_response(rows, cols, data)) == ref.response_capacity(rows, cols, ct)
            data = [int(v) for v in rng.integers(0, 1 << ct, size=rows * cols, dtype=np.uint64)]
            assert len(ref.encode_response(rows, cols, data)) <= ref.response_capacity(rows, cols, ct)


# ---- google.protobuf

def protobuf_classes():
    pytest.importorskip("google.protobuf")
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    F = descriptor_pb2.FieldDescriptorProto
    fd = descriptor_pb2.FileDescriptorProto(name="simple_pir_proto_test.proto", package="t", syntax="proto3")
    one, rep = F.LABEL_OPTIONAL, F.LABEL_REPEATED

    def msg(name, fields):
        m = fd.message_type.add(name=name)
        for number, fname, ftype, label, type_name in fields:
            f = m.field.add(name=fname, number=number, type=ftype, label=label)
            if type_name:
                f.type_name = ".t." + type_name
        return m

    msg("SimplePIRMatrix", [(1, "row_count", F.TYPE_UINT32, one, None), (2, "col_count", F.TYPE_UINT32, one, None),
                            (3, "data", F.TYPE_UINT64, rep, None)])
    msg("SimplePIRRequest", [(1, "request", F.TYPE_MESSAGE, one, "SimplePIRMatrix"), (2, "shard_index", F.TYPE_UINT32, one, None),
                             (3, "configuration_hash", F.TYPE_BYTES, one, None)])
    msg("SimplePIRResponse", [(1, "response", F.TYPE_MESSAGE, one, "SimplePIRMatrix")])
    msg("SimplePIREncryptionParams", [(1, "lattice_dimension", F.TYPE_UINT32, one, None),
                                      (2, "error_std_dev", F.TYPE_DOUBLE, one, None),
                                      (3, "plaintext_bits", F.TYPE_UINT32, one, None),
                                      (4, "ciphertext_bits", F.TYPE_UINT32, one, None)])
    msg("SimplePIRParameters", [(1, "encryption_params", F.TYPE_MESSAGE, one, "SimplePIREncryptionParams"),
                                (2, "a_seed", F.TYPE_BYTES, one, None), (3, "entry_size_in_bytes", F.TYPE_UINT32, one, None),
                                (4, "entries_per_column", F.TYPE_UINT32, one, None),
                                (5, "chunks_per_entry", F.TYPE_UINT32, one, None),
                                (6, "database_columns", F.TYPE_UINT32, one, None)])
    msg("ChunkLocation", [(1, "shard_index", F.TYPE_UINT32, one, None), (2, "index", F.TYPE_UINT32, one, None)])
    msg("Entry", [(1, "original_index", F.TYPE_UINT64, one, None), (2, "size", F.TYPE_UINT32, one, None),
                  (3, "chunks", F.TYPE_MESSAGE, rep, "ChunkLocation")])
    msg("DatabaseMapping", [(1, "entries", F.TYPE_MESSAGE, rep, "Entry"), (2, "chunk_size", F.TYPE_UINT32, one, None)])
    msg("SimplePIRConfig", [(1, "database_mapping", F.TYPE_MESSAGE, one, "DatabaseMapping"),
                            (2, "params", F.TYPE_MESSAGE, rep, "SimplePIRParameters"),
                            (3, "hint_identifiers", F.TYPE_BYTES, rep, None)])
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    return {n: message_factory.GetMessageClass(pool.FindMessageTypeByName("t." + n))
            for n in ["SimplePIRRequest", "SimplePIRResponse", "SimplePIRConfig"]}


DATA_FORMS = {
    "packed": lambda v: ref.packed(3, v),
    "split": lambda v: ref.split_packed(3, v, [1, 3, 6]),
    "unpacked": lambda v: ref.unpacked(3, v),
}


@pytest.mark.parametrize("form", sorted(DATA_FORMS))
def test_protobuf_parses_the_restatement(form):
    cls = protobuf_classes()
    data = ref.encode_request_with(2, 4, DATA_FORMS[form](VALUES), 5)
    m = cls["SimplePIRRequest"]()
    m.ParseFromString(data)
    assert (m.request.row_count, m.request.col_count, list(m.request.data), m.shard_index) == (2, 4, VALUES, 5)
    assert ref.parse_request(data) == ((2, 4, VALUES), 5, b"")


def test_protobuf_writes_the_restatements_bytes():
    cls = protobuf_classes()
    for rows, cols, data in ((2, 4, VALUES), (0, 7, []), (1, 1, [0])):
        m = cls["SimplePIRResponse"]()
        m.response.row_count, m.response.col_count = rows, cols
        m.response.data.extend(data)
        m.response.SetInParent()
        assert m.SerializeToString(deterministic=True) == ref.encode_response(rows, cols, data)
        r = cls["SimplePIRRequest"]()
        r.request.row_count, r.request.col_count, r.shard_index, r.configuration_hash = rows, cols, 3, b"xy"
        r.request.data.extend(data)
        r.request.SetInParent()
        assert r.SerializeToString(deterministic=True) == ref.encode_request(rows, cols, data, 3, b"xy")
    c = cls["SimplePIRConfig"]()
    c.database_mapping.chunk_size = 30
    e = c.database_mapping.entries.add(original_index=5, size=100)
    e.chunks.add(shard_index=0, index=1)
    e.chunks.add(shard_index=1, index=0)
    p = c.params.add(a_seed=SEED, entry_size_in_bytes=52, entries_per_column=1, chunks_per_entry=5, database_columns=1000)
    p.encryption_params.lattice_dimension, p.encryption_params.error_std_dev = 2048, 6.4
    p.encryption_params.plaintext_bits, p.encryption_params.ciphertext_bits = 14, 42
    c.hint_identifiers.extend([b"a" * 32, b""])
    assert c.SerializeToString(deterministic=True) == ref.encode_config(
        [(5, 100, [(0, 1), (1, 0)])], 30, [(2048, 6.4, 14, 42, SEED, 52, 1, 5, 1000)], [b"a" * 32, b""])


# ---- the library's host-only calls

def lib_ok():
    try:
        hecuda.load_library()
    except hecuda.HeError:
        pytest.skip("libhecuda.so is not built")


def test_library_request_writer_and_walk():
    lib_ok()
    words = np.array(VALUES, np.uint64).reshape(2, 4)
    msg = sp.SimplePirRequest.write(words, 3, b"hash")
    assert msg == ref.encode_request(2, 4, VALUES, 3, b"hash")
    f = sp.SimplePirRequest.fields(msg)
    assert (f["row_count"], f["col_count"], f["shard_index"], f["configuration_hash"], f["data_run_count"]) == (2, 4, 3, b"hash", 1)
    for form, runs in (("split", 4), ("unpacked", 8)):
        f = sp.SimplePirRequest.fields(ref.encode_request_with(2, 4, DATA_FORMS[form](VALUES), 1))
        assert (f["data_run_count"], f["shard_index"]) == (runs, 1)
    assert sp.SimplePirRequest.fields(ref.field_scalar(2, 1))["has_request"] is False
    # uint32 fields keep their low 32 bits
    f = sp.SimplePirRequest.fields(ref.field_bytes(1, ref.field_scalar(1, (1 << 32) + 3)))
    assert f["row_count"] == 3


@pytest.mark.parametrize("bad,what", [
    (b"\x0a\x05\x08", "truncated"),
    (ref.field_bytes(1, b"") * 2, "given twice"),
    (ref.field_bytes(1, ref.varint(3 << 3 | 5) + b"\0\0\0\0"), "wire type 5"),
    (ref.field_bytes(1, ref.varint(1 << 3 | 3)), "groups"),
    (b"\x10" + b"\x80" * 10 + b"\x01", "longer than 10"),
])
def test_library_request_walk_refusals(bad, what):
    lib_ok()
    with pytest.raises(hecuda.HeError, match=what):
        sp.SimplePirRequest.fields(bad)


def test_library_response_reader():
    lib_ok()
    for rows, cols, data in ((2, 4, VALUES), (0, 7, [])):
        for form in DATA_FORMS.values():
            msg = ref.field_bytes(1, ref.field_scalar(1, rows) + ref.field_scalar(2, cols) + (form(data) if data else b""))
            assert np.array_equal(sp.SimplePirResponse.read(msg), np.array(data, np.uint64).reshape(rows, cols))
    with pytest.raises(hecuda.HeError, match="values for"):
        sp.SimplePirResponse.read(ref.encode_response(2, 4, VALUES[:7]))
    with pytest.raises(sp.PirError, match="2\\^32"):
        sp.SimplePirResponse.read(ref.encode_response(2, 4, VALUES), np.uint32)


def sample_config(ct=42, std=6.4, seed=SEED):
    entries = [(5, 100, [(0, 1), (1, 0), (0, 0), (1, 1)]), (9, 60, [(0, 2), (1, 2)])]
    params = [(2048, std, 14, ct, seed, 30, 1, 5, 15), (2048, std, 14, ct, seed[::-1], 30, 1, 5, 15)]
    return entries, params


def test_library_config_round_trip():
    lib_ok()
    entries, params = sample_config()
    raw = ref.encode_config(entries, 30, params, [b"a" * 32, b"b" * 32])
    cfg = sp.SimplePirConfig.deserialize(raw)
    assert cfg.serialize() == raw
    assert cfg.scalar == np.uint64
    assert cfg.databaseMap.chunkSize == 30 and list(cfg.databaseMap.originalIndices) == [5, 9]
    assert cfg.params[1].seed == SEED[::-1] and cfg.params[0].databaseColumns == 15
    assert cfg.params[0].encryptionParams.errorStdDev == 6.4
    assert sp.SimplePirConfig.deserialize(ref.encode_config(*[sample_config(ct=28, std=3.2)[0], 30,
                                                              sample_config(ct=28, std=3.2)[1], []])).scalar == np.uint32


@pytest.mark.parametrize("params,what", [
    ([(2048, 5.0, 14, 42, SEED, 30, 1, 5, 15)], "errorStdDev"),
    ([(2048, 6.4, 14, 42, SEED[:31], 30, 1, 5, 15)], "a_seed of 31 bytes"),
    ([(2048, 6.4, 14, 42, b"", 30, 1, 5, 15)], "a_seed of 0 bytes"),
    ([(2000, 6.4, 14, 42, SEED, 30, 1, 5, 15)], "power of 2"),
    ([(2048, 6.4, 14, 32, SEED, 30, 1, 5, 15)], "scalar width"),  # ct 32 -> 32-bit words, ct + 1 > 32
    ([(2048, 6.4, 14, 42, SEED, 30, 2, 5, 15)], "entriesPerColumn"),
])
def test_library_config_refusals(params, what):
    lib_ok()
    with pytest.raises(hecuda.HeError, match=what):
        sp.SimplePirConfig.deserialize(ref.encode_config(sample_config()[0], 30, params, []))


# ---- the device maps on the CPU

@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    binary = str(tmp_path_factory.mktemp("emu") / "simple_pir_proto_emulate")
    subprocess.check_call([NVCC, "-O1", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", binary, EMU_SRC])

    def run(args, data):
        out = subprocess.run([binary] + [str(a) for a in args], input=(data.hex() or ".") + "\n", capture_output=True,
                             text=True, check=True).stdout
        return out.strip().splitlines()
    return run


def emu_decode(emu, message, columns, row_base, col_tiles, ct, word32):
    lines = emu(["decode", columns, row_base, col_tiles, ct, int(word32)], message)
    if lines[0].startswith("error"):
        return lines[0]
    flags = int(lines[0].split()[1])
    return flags, [tuple(int(x) for x in line.split()) for line in lines[1:]]


@pytest.mark.parametrize("form", sorted(DATA_FORMS))
def test_emulated_decode_places_every_digit(emu, form):
    rng = np.random.default_rng(len(form))
    for ct, word32 in ((28, True), (42, False), (61, False)):
        rows, cols = 3, 45
        top = (1 << 32) - 1 if word32 else (1 << 64) - 1
        values = [int(v) for v in rng.integers(0, top, size=rows * cols, dtype=np.uint64, endpoint=True)]
        values[:5] = [0, 127, 128, 1 << 28, (1 << 32) - 1]
        col_tiles, row_base = 2, 5
        got = emu_decode(emu, ref.encode_request_with(rows, cols, DATA_FORMS[form](values)), cols, row_base, col_tiles,
                         ct, word32)
        assert got[0] == 0
        want = []
        for i, v in enumerate(values):
            at = ref.b_offset(row_base + i // cols, i % cols, col_tiles)
            want.append((at, v & ((1 << ct) - 1)))
        assert sorted(got[1]) == sorted(want)


@pytest.mark.parametrize("data,flag", [
    (b"\x01\x85", 2),                                 # runs past its run
    (b"\x01" + b"\x80" * 10 + b"\x01", 1),            # longer than 10 bytes
    (b"\x01" + b"\xff" * 9 + b"\x01", 4),             # 2^63 + ... on a 32-bit shard
    (b"\x01\x02\x03", 8),                             # three values for 1 x 2
])
def test_emulated_decode_flags(emu, data, flag):
    got = emu_decode(emu, ref.encode_request_with(1, 2, ref.field_bytes(3, data)), 2, 0, 1, 28, True)
    assert got[0] & flag


def test_emulated_decode_accepts_what_read_varint_accepts(emu):
    ten = b"\xff" * 9 + b"\x01"  # ten bytes, 2^64 - 1
    got = emu_decode(emu, ref.encode_request_with(1, 2, ref.field_bytes(3, b"\x00" + ten)), 2, 0, 1, 61, False)
    assert got[0] == 0 and sorted(v for _, v in got[1]) == [0, (1 << 61) - 1]


def test_emulated_encode_gives_the_restatements_bytes(emu):
    rng = np.random.default_rng(4)
    for ct in (28, 32, 42, 61):
        for rows, cols in ((0, 5), (1, 1), (3, 37)):
            acc = [int(v) for v in rng.integers(0, 1 << 64, size=rows * cols, dtype=np.uint64, endpoint=False)]
            out = emu(["encode", rows, cols, ct] + acc, b"")
            mask = (1 << ct) - 1
            want = ref.encode_response(rows, cols, [v & mask for v in acc])
            assert bytes.fromhex(out[0] if out and out[0] != "." else "") == want
            assert int(out[1]) == ref.response_capacity(rows, cols, ct)
