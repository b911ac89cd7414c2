"""Processed PNNS databases in the reference's protobuf format, on the CPU.

- A known-answer test pins the restatement (tests/pnns_database_io_ref.py) with bytes written out by hand.
- A cross-check against google.protobuf, with descriptors built here from the .proto field tables: it parses the
  restatement's bytes to the same values, and a message it builds serializes to the restatement's bytes.  This stands
  in for bytes written by SwiftProtobuf, which cannot be produced here; both follow the same proto3 encoding rules.
- tests/emu/pnns_database_io_emulate.cu runs the library's own walker, writer and chunk planner (pnns_database_io.hpp,
  database_io.hpp) on the CPU and must reproduce the restatement: the same plaintext offsets, entries and config on
  load, the same bytes on save, and the same refusals."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import pnns_database_io_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_SRC = os.path.join(ROOT, "tests", "emu", "pnns_database_io_emulate.cu")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"

# N = 16, t = 17 and one extra plaintext modulus 113, moduli [97, 193]; 3 x 2 vectors: two plaintexts per matrix
KAT_CONFIG = {
    "client_config": {
        "encryption_parameters": {"polynomial_degree": 16, "plaintext_modulus": 17, "coefficient_moduli": [97, 193],
                                  "he_scheme": 1},
        "scaling_factor": 100, "query_packing": ("denseRow",), "vector_dimension": 2, "galois_elements": [31, 3],
        "extra_plaintext_moduli": [113]},
    "database_packing": ("diagonal", (2, 2, 1)),
}
KAT_MATRICES = [
    {"num_rows": 3, "num_columns": 2, "plaintexts": [b"\xaa\xbb", b"\xcc\xdd"], "packing": ("diagonal", (2, 2, 1))},
    {"num_rows": 3, "num_columns": 2, "plaintexts": [b"\x01\x02", b"\x03\x04"], "packing": ("diagonal", (2, 2, 1))},
]
KAT_IDS = [1, 300, 5]
KAT_METADATA = [b"a", b"", b"xyz"]
PACKING = "12081206" "080210021801"  # diagonal { baby_step_giant_step { 2, 2, 1 } }
KAT_BYTES = bytes.fromhex(
    "0a1c" "0803" "1002" "1a040a02aabb" "1a040a02ccdd" "220a" + PACKING +
    "0a1c" "0803" "1002" "1a040a020102" "1a040a020304" "220a" + PACKING +
    "120401ac0205" "1a0161" "1a00" "1a0378797a"
    "222a" "0a1c" "0a0b" "0810" "1011" "1a0361c101" "3001" "1064" "1a020a00" "2002" "2a021f03" "3a0171"
    "120a" + PACKING)


def test_known_answer():
    data = ref.encode_processed_database(KAT_MATRICES, KAT_IDS, KAT_METADATA, KAT_CONFIG)
    assert data == KAT_BYTES, data.hex()
    parsed = ref.parse_processed_database(KAT_BYTES)
    assert [m["plaintexts"] for m in parsed["matrices"]] == [m["plaintexts"] for m in KAT_MATRICES]
    assert parsed["entry_ids"] == KAT_IDS and parsed["entry_metadatas"] == KAT_METADATA
    c = parsed["server_config"]
    assert c["database_packing"] == ("diagonal", (2, 2, 1))
    assert c["client_config"]["extra_plaintext_moduli"] == [113]
    assert c["client_config"]["encryption_parameters"]["coefficient_moduli"] == [97, 193]


# ---- google.protobuf -------------------------------------------------------------------------------------------------

def protobuf_classes():
    pytest.importorskip("google.protobuf")
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    F = descriptor_pb2.FieldDescriptorProto
    fd = descriptor_pb2.FileDescriptorProto(name="pnns_test.proto", package="t", syntax="proto3")

    def msg(name, fields, oneof=None):
        m = fd.message_type.add(name=name)
        if oneof:
            m.oneof_decl.add(name=oneof)
        for number, fname, ftype, label, type_name in fields:
            f = m.field.add(name=fname, number=number, type=ftype, label=label)
            if type_name:
                f.type_name = ".t." + type_name
            if oneof:
                f.oneof_index = 0

    one, rep = F.LABEL_OPTIONAL, F.LABEL_REPEATED
    msg("EncryptionParameters", [(1, "polynomial_degree", F.TYPE_UINT64, one, None),
                                 (2, "plaintext_modulus", F.TYPE_UINT64, one, None),
                                 (3, "coefficient_moduli", F.TYPE_UINT64, rep, None),
                                 (4, "error_std_dev", F.TYPE_INT32, one, None),
                                 (5, "security_level", F.TYPE_INT32, one, None),
                                 (6, "he_scheme", F.TYPE_INT32, one, None)])
    msg("BabyStepGiantStep", [(1, "vector_dimension", F.TYPE_UINT32, one, None), (2, "baby_step", F.TYPE_UINT32, one, None),
                              (3, "giant_step", F.TYPE_UINT32, one, None)])
    msg("Empty", [])
    msg("Diagonal", [(2, "baby_step_giant_step", F.TYPE_MESSAGE, one, "BabyStepGiantStep")])
    msg("MatrixPacking", [(1, "dense_row", F.TYPE_MESSAGE, one, "Empty"), (2, "diagonal", F.TYPE_MESSAGE, one, "Diagonal"),
                          (3, "dense_column", F.TYPE_MESSAGE, one, "Empty")], oneof="matrix_packing_type")
    msg("ClientConfig", [(1, "encryption_parameters", F.TYPE_MESSAGE, one, "EncryptionParameters"),
                         (2, "scaling_factor", F.TYPE_UINT64, one, None), (3, "query_packing", F.TYPE_MESSAGE, one, "MatrixPacking"),
                         (4, "vector_dimension", F.TYPE_UINT32, one, None), (5, "galois_elements", F.TYPE_UINT32, rep, None),
                         (6, "distance_metric", F.TYPE_INT32, one, None),
                         (7, "extra_plaintext_moduli", F.TYPE_UINT64, rep, None)])
    msg("ServerConfig", [(1, "client_config", F.TYPE_MESSAGE, one, "ClientConfig"),
                         (2, "database_packing", F.TYPE_MESSAGE, one, "MatrixPacking")])
    msg("SerializedPlaintext", [(1, "poly", F.TYPE_BYTES, one, None)])
    msg("SerializedPlaintextMatrix", [(1, "num_rows", F.TYPE_UINT32, one, None), (2, "num_columns", F.TYPE_UINT32, one, None),
                                      (3, "plaintexts", F.TYPE_MESSAGE, rep, "SerializedPlaintext"),
                                      (4, "packing", F.TYPE_MESSAGE, one, "MatrixPacking")])
    msg("SerializedProcessedDatabase", [(1, "plaintext_matrices", F.TYPE_MESSAGE, rep, "SerializedPlaintextMatrix"),
                                        (2, "entry_ids", F.TYPE_UINT64, rep, None),
                                        (3, "entry_metadatas", F.TYPE_BYTES, rep, None),
                                        (4, "server_config", F.TYPE_MESSAGE, one, "ServerConfig")])
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    return {name: message_factory.GetMessageClass(pool.FindMessageTypeByName("t." + name))
            for name in ("SerializedProcessedDatabase", "ServerConfig", "ClientConfig")}


def fill_packing(p, packing):
    if packing[0] == "diagonal":
        d, b, g = packing[1]
        p.diagonal.baby_step_giant_step.vector_dimension, p.diagonal.baby_step_giant_step.baby_step = d, b
        p.diagonal.baby_step_giant_step.giant_step = g
    elif packing[0] == "denseRow":
        p.dense_row.SetInParent()
    else:
        p.dense_column.SetInParent()


def fill_client(c, cfg):
    e = cfg["encryption_parameters"]
    c.encryption_parameters.polynomial_degree, c.encryption_parameters.plaintext_modulus = e["polynomial_degree"], e["plaintext_modulus"]
    c.encryption_parameters.coefficient_moduli.extend(e["coefficient_moduli"])
    c.encryption_parameters.error_std_dev = e.get("error_std_dev", 0)
    c.encryption_parameters.security_level = e.get("security_level", 0)
    c.encryption_parameters.he_scheme = e.get("he_scheme", 1)
    c.scaling_factor, c.vector_dimension = cfg["scaling_factor"], cfg["vector_dimension"]
    fill_packing(c.query_packing, cfg["query_packing"])
    c.galois_elements.extend(cfg.get("galois_elements", []))
    c.extra_plaintext_moduli.extend(cfg.get("extra_plaintext_moduli", []))


def test_google_protobuf_agrees_with_the_restatement():
    classes = protobuf_classes()
    db = classes["SerializedProcessedDatabase"]()
    for m in KAT_MATRICES:
        pm = db.plaintext_matrices.add(num_rows=m["num_rows"], num_columns=m["num_columns"])
        for poly in m["plaintexts"]:
            pm.plaintexts.add(poly=poly)
        fill_packing(pm.packing, m["packing"])
    db.entry_ids.extend(KAT_IDS)
    db.entry_metadatas.extend(KAT_METADATA)
    fill_client(db.server_config.client_config, KAT_CONFIG["client_config"])
    fill_packing(db.server_config.database_packing, KAT_CONFIG["database_packing"])
    assert db.SerializeToString() == KAT_BYTES
    parsed = classes["SerializedProcessedDatabase"].FromString(KAT_BYTES)
    assert parsed == db
    assert list(parsed.entry_ids) == KAT_IDS and [bytes(m) for m in parsed.entry_metadatas] == KAT_METADATA
    # the configs on their own, and one with a .diagonal query packing, stdDev64 and quantum128
    cfg = dict(KAT_CONFIG["client_config"], query_packing=("diagonal", (4, 2, 2)),
               encryption_parameters=dict(KAT_CONFIG["client_config"]["encryption_parameters"], error_std_dev=1,
                                          security_level=1))
    client = classes["ClientConfig"]()
    fill_client(client, cfg)
    assert client.SerializeToString() == ref.encode_client_config(cfg)
    server = classes["ServerConfig"]()
    fill_client(server.client_config, cfg)
    fill_packing(server.database_packing, ("diagonal", (8, 3, 3)))
    data = ref.encode_server_config({"client_config": cfg, "database_packing": ("diagonal", (8, 3, 3))})
    assert server.SerializeToString() == data
    assert ref.parse_server_config(data)["client_config"]["query_packing"] == ("diagonal", (4, 2, 2))


# ---- the library's walker and writer, replayed on the CPU -------------------------------------------------------------

@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    binary = str(tmp_path_factory.mktemp("emu") / "pnns_database_io_emulate")
    subprocess.check_call([NVCC, "-O1", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", binary, EMU_SRC])
    return binary


def run(binary, args, data: bytes):
    return subprocess.run([binary] + args, input=(data.hex() or ".") + "\n", capture_output=True, text=True,
                          check=True).stdout.splitlines()


def config_line(cfg: dict) -> str:
    c, e = cfg["client_config"], cfg["client_config"]["encryption_parameters"]
    q, d = c["query_packing"], cfg.get("database_packing", ("none",))
    kinds = {"none": 0, **ref.PACKINGS}
    values = [e["polynomial_degree"], e["plaintext_modulus"], len(e["coefficient_moduli"]), *e["coefficient_moduli"],
              e.get("error_std_dev", 0), e.get("security_level", 0), e.get("he_scheme", 0), c["scaling_factor"],
              kinds[q[0]], *(q[1] if len(q) > 1 else (0, 0, 0)), c["vector_dimension"], len(c["galois_elements"]),
              *c["galois_elements"], c.get("distance_metric", 0), len(c["extra_plaintext_moduli"]),
              *c["extra_plaintext_moduli"], kinds[d[0]], *(d[1] if len(d) > 1 else (0, 0, 0))]
    return "config " + " ".join(str(v) for v in values)


def random_database(seed, matrices=2, count=6, poly_bytes=40, metadata=True):
    rng = np.random.default_rng(seed)
    ms = [{"num_rows": 70, "num_columns": 5, "packing": ("diagonal", (8, 3, 3)),
           "plaintexts": [rng.integers(0, 256, poly_bytes, dtype=np.uint8).tobytes() for _ in range(count)]}
          for _ in range(matrices)]
    ids = [int(v) for v in rng.integers(0, 1 << 63, 70, dtype=np.uint64)] + [(1 << 64) - 1]
    meta = [rng.integers(0, 256, int(rng.integers(0, 5)), dtype=np.uint8).tobytes() for _ in ids] if metadata else []
    cfg = {"client_config": dict(KAT_CONFIG["client_config"], extra_plaintext_moduli=[113] * (matrices - 1)),
           "database_packing": ("diagonal", (8, 3, 3))}
    return ms, ids, meta, cfg


@pytest.mark.parametrize("matrices,metadata", [(1, False), (2, True), (3, True)])
def test_walk_and_resave_reproduce_the_restatement(emu, matrices, metadata):
    ms, ids, meta, cfg = random_database(matrices, matrices, metadata=metadata)
    data = ref.encode_processed_database(ms, ids, meta, cfg)
    lines = run(emu, ["walk"], data)
    assert lines[0] == "ok"
    for k, m in enumerate(ms):
        assert lines[1 + 2 * k] == f"matrix 70 5 2 8 3 3 {len(m['plaintexts'])}"
        polys = [tuple(int(v) for v in item.split(":")) for item in lines[2 + 2 * k].split()[1:]]
        assert [data[a:a + b] for a, b in polys] == m["plaintexts"]
    rest = lines[1 + 2 * len(ms):]
    assert [int(v) for v in rest[0].split()[1:]] == ids
    metas = [tuple(int(v) for v in item.split(":")) for item in rest[1].split()[1:]]
    assert [data[a:a + b] for a, b in metas] == meta
    assert rest[2] == config_line(cfg)
    poly = 40 + 8  # a plaintext and its framing
    for budget in (poly // 2, 2 * poly, 3 * poly + 1, len(data)):
        out = run(emu, ["resave", str(budget)], data)
        assert bytes.fromhex(out[1]) == data
        per_matrix = 6 if budget < 2 * poly else -(-6 // (budget // poly)) if budget < len(data) else 1
        assert int(out[0].split()[1]) == matrices * per_matrix


def test_walk_accepts_any_conforming_encoding(emu):
    ms, ids, meta, cfg = random_database(7, 2)
    data = ref.encode_processed_database(ms, ids, meta, cfg)
    expected = run(emu, ["walk"], data)
    ids_line = expected[5]
    fields = list(ref.fields(data))

    def field_bytes(number, wire, v):
        if wire == 0:
            return ref.key(number, 0) + ref.varint(v)
        return ref.message(number, v)

    # fields out of order (the config first, then entries, then the matrices), unknown fields of every skippable type
    unknown = ref.key(9, 0) + ref.varint(5) + ref.key(10, 1) + bytes(8) + ref.message(11, b"xyz") + ref.key(12, 5) + bytes(4)
    shuffled = b"".join(field_bytes(*f) for f in reversed(fields)) + unknown
    lines = run(emu, ["walk"], shuffled)
    assert lines[0] == "ok" and lines[5] == ids_line and lines[-1] == expected[-1]
    # unpacked entry ids
    unpacked = b"".join(field_bytes(*f) for f in fields if f[0] != 2) + b"".join(ref.scalar(2, v) if v else ref.key(2, 0) + b"\0" for v in ids)
    lines = run(emu, ["walk"], unpacked)
    assert lines[0] == "ok" and lines[5] == ids_line


def test_walk_refuses_what_the_reference_refuses(emu):
    ms, ids, meta, cfg = random_database(3, 1, count=2, poly_bytes=3)
    data = ref.encode_processed_database(ms, ids, meta, cfg)
    # truncation at every framing byte: cutting the file anywhere refuses it (the config comes last)
    for end in range(len(data)):
        assert run(emu, ["walk"], data[:end])[0].startswith("error -1"), end
    refusals = {
        "wire type": ref.key(1, 0) + ref.varint(3) + data,                         # a matrix given as a varint
        "varint longer than 10 bytes": data + ref.key(9, 0) + b"\xff" * 10 + b"\x01",
        "groups": data + ref.key(9, 3),
        "unsetField(SerializedProcessedDatabase.serverConfig)": b"".join(ref.message(1, f[2]) for f in ref.fields(data)
                                                                          if f[0] == 1),
        "given twice": data + ref.message(4, ref.encode_server_config(cfg)),
    }
    for what, raw in refusals.items():
        line = run(emu, ["walk"], raw)[0]
        assert line.startswith("error -1") and what in line, (what, line)


def config_refusal(emu, mode, cfg_bytes):
    return run(emu, [mode], cfg_bytes)[0]


def test_config_round_trips_and_refusals(emu):
    cfg = {"client_config": dict(KAT_CONFIG["client_config"], query_packing=("diagonal", (4, 2, 2)),
                                 encryption_parameters=dict(KAT_CONFIG["client_config"]["encryption_parameters"],
                                                            error_std_dev=1, security_level=1)),
           "database_packing": ("denseColumn",)}
    data = ref.encode_server_config(cfg)
    lines = run(emu, ["server"], data)
    assert lines[0] == config_line(cfg) and bytes.fromhex(lines[1]) == data
    client = ref.encode_client_config(cfg["client_config"])
    lines = run(emu, ["client"], client)
    assert lines[0] == config_line({"client_config": cfg["client_config"]}) and bytes.fromhex(lines[1]) == client
    e = cfg["client_config"]["encryption_parameters"]
    cases = {
        "unsetField(ServerConfig.clientConfig)": ref.message(2, ref.encode_packing(("denseRow",))),
        "unsetField(ClientConfig.encryptionParameters)":
            ref.message(1, ref.scalar(2, 5) + ref.message(3, ref.encode_packing(("denseRow",)))),
        "invalidScheme": ref.message(1, ref.encode_client_config(dict(cfg["client_config"],
                                                                      encryption_parameters=dict(e, he_scheme=2)))),
        "unrecognizedEnumValue(enum: ErrorStdDev, value: 7)":
            ref.message(1, ref.encode_client_config(dict(cfg["client_config"], encryption_parameters=dict(e, error_std_dev=7)))),
        "unrecognizedEnumValue(enum: DistanceMetric, value: 1)":
            ref.message(1, ref.encode_client_config(dict(cfg["client_config"], distance_metric=1))),
        "unsetOneof(MatrixPacking.matrixPackingType)": ref.message(1, ref.encode_client_config(cfg["client_config"])),
    }
    for what, raw in cases.items():
        line = config_refusal(emu, "server", raw)
        assert line.startswith("error -1") and what in line, (what, line)
    with pytest.raises(ref.ProtoError, match="invalidScheme"):
        ref.parse_server_config(cases["invalidScheme"])
    # more moduli than the struct holds: unsupported
    big = dict(cfg["client_config"], encryption_parameters=dict(e, coefficient_moduli=list(range(3, 3 + 2 * 33, 2))))
    line = config_refusal(emu, "client", ref.encode_client_config(big))
    assert line.startswith("error -2"), line
