"""PNNS requests and responses in the reference's protobuf messages, and the query plan, on the CPU.

- Known-answer byte strings, written out by hand at N = 16, pin the restatement (tests/pnns_proto_ref.py) for
  PNNSRequest (one and two query matrices, with and without evaluation_key) and PNNSShardResponse (one and two reply
  matrices; absent, empty and non-empty metadata).
- A cross-check against google.protobuf, with descriptors built here from the .proto field tables: it parses the
  restatement's bytes to the same values, and messages it builds serialize to the restatement's bytes.
- tests/emu/pnns_proto_emulate.cu runs the library's own walks, refusals and response template (pnns_proto.hpp) on the
  CPU and must reproduce the restatement; it runs the library's query plan (pnns_plan.hpp) over a sweep of shapes and
  Galois sets, and must give what PlaintextMatrix._rowDescriptors derives in Python."""
import os
import random
import shutil
import subprocess
import sys

import pytest

import pir_proto_ref as pref
import pnns_proto_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "swift-homomorphic-encryption_b200"))
from hecuda import pnns  # noqa: E402  (host-only: CiphertextMatrix, GaloisElement)

EMU_SRC = os.path.join(ROOT, "tests", "emu", "pnns_proto_emulate.cu")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ERR_INVALID = -1

# N = 16 over rows of 5 and 6 bits: a poly0 is 10 + 12 = 22 bytes; a reply row of 5 bits with skip_lsbs [1, 2] is 8 + 6
N, BITS = 16, [5, 6]
SIZES = pref.poly_sizes(N, BITS)
POLY0, SEED = bytes(range(22)), bytes(range(32, 64))
SEEDED = ("seeded", POLY0, SEED)
CT_HEX = "0a3a" "0a16" + POLY0.hex() + "1220" + SEED.hex()  # SerializedCiphertext { seeded { poly0 seed } }
MATRIX_HEX = "0801" "1002" "1a3c" + CT_HEX + "2202" "0a00"  # 1 x 2, one ciphertext, .denseRow
KAT_REQUEST_1 = bytes.fromhex("1246" + MATRIX_HEX)
KAT_REQUEST_2 = bytes.fromhex("1246" + MATRIX_HEX + "1246" + MATRIX_HEX)
KEY = bytes.fromhex("abcd")
KAT_REQUEST_KEY = bytes.fromhex("0a020307" "1246" + MATRIX_HEX + "220109" "2a0c" "0a06" "0805" "12026b30" "1202abcd"
                                "32017a")
P0, P1 = bytes(range(100, 108)), bytes(range(200, 206))
FULL_HEX = "1218" "0a10" "0200" + P0.hex() + P1.hex() + "12020102" "1801"  # SerializedCiphertext { full }
REPLY_HEX = "0a24" "0803" "1001" "1a1a" + FULL_HEX + "2202" "1a00"  # 3 x 1, one reply, .denseColumn
KAT_RESPONSE_1 = bytes.fromhex(REPLY_HEX + "1203070809")
KAT_RESPONSE_2 = bytes.fromhex(REPLY_HEX + REPLY_HEX + "1203070809" "1a01aa" "1a00" "1a02bbcc")


def test_known_answers():
    matrix = ref.encode_matrix(1, 2, [SEEDED], ref.DENSE_ROW)
    assert matrix == bytes.fromhex(MATRIX_HEX)
    assert ref.encode_pnns_request([matrix]) == KAT_REQUEST_1
    assert ref.encode_pnns_request([matrix, matrix]) == KAT_REQUEST_2
    assert ref.encode_pnns_request([matrix], shard_indices=[3, 7], config_id=b"\x09", evaluation_key=KEY,
                                   key_metadata=(5, b"k0"), shard_ids=["z"]) == KAT_REQUEST_KEY
    fields = ref.parse_pnns_request(KAT_REQUEST_KEY)
    assert (fields["shardIndices"], fields["configId"], fields["shardIds"]) == ([3, 7], b"\x09", ["z"])
    assert (fields["keyTimestamp"], fields["keyIdentifier"]) == (5, b"k0")
    assert KAT_REQUEST_KEY[fields["evaluationKey"][0]:fields["evaluationKey"][1]] == KEY
    assert ref.parse_matrix(KAT_REQUEST_1, *ref.parse_pnns_request(KAT_REQUEST_1)["query"][0], SIZES) == \
        (1, 2, ref.DENSE_ROW, [SEEDED])
    one = ([(P0, P1)], [1, 2])
    assert ref.encode_shard_response([one], 3, 1, [7, 8, 9], []) == KAT_RESPONSE_1
    assert ref.encode_shard_response([one, one], 3, 1, [7, 8, 9], [b"\xaa", b"", b"\xbb\xcc"]) == KAT_RESPONSE_2
    matrices, ids, metadata = ref.parse_shard_response(KAT_RESPONSE_2, pref.poly_sizes(N, [5]))
    assert ids == [7, 8, 9] and metadata == [b"\xaa", b"", b"\xbb\xcc"]
    assert matrices[1] == (3, 1, ref.DENSE_COLUMN, [("full", b"\x02\x00" + P0 + P1, [1, 2], 1)])


# ---- google.protobuf -------------------------------------------------------------------------------------------------

def protobuf_classes():
    pytest.importorskip("google.protobuf")
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    F = descriptor_pb2.FieldDescriptorProto
    fd = descriptor_pb2.FileDescriptorProto(name="pnns_proto_test.proto", package="t", syntax="proto3")
    one, rep = F.LABEL_OPTIONAL, F.LABEL_REPEATED

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
        return m

    msg("SerializedSeededCiphertext", [(1, "poly0", F.TYPE_BYTES, one, None), (2, "seed", F.TYPE_BYTES, one, None)])
    msg("SerializedFullCiphertext", [(1, "polys", F.TYPE_BYTES, one, None), (2, "skip_lsbs", F.TYPE_UINT32, rep, None),
                                     (3, "correction_factor", F.TYPE_UINT64, one, None)])
    msg("SerializedCiphertext", [(1, "seeded", F.TYPE_MESSAGE, one, "SerializedSeededCiphertext"),
                                 (2, "full", F.TYPE_MESSAGE, one, "SerializedFullCiphertext")], oneof="type")
    msg("Empty", [])
    msg("BabyStepGiantStep", [(1, "vector_dimension", F.TYPE_UINT32, one, None), (2, "baby_step", F.TYPE_UINT32, one, None),
                              (3, "giant_step", F.TYPE_UINT32, one, None)])
    msg("MatrixPackingDiagonal", [(2, "baby_step_giant_step", F.TYPE_MESSAGE, one, "BabyStepGiantStep")])
    msg("MatrixPacking", [(1, "dense_row", F.TYPE_MESSAGE, one, "Empty"),
                          (2, "diagonal", F.TYPE_MESSAGE, one, "MatrixPackingDiagonal"),
                          (3, "dense_column", F.TYPE_MESSAGE, one, "Empty")], oneof="matrix_packing_type")
    msg("SerializedCiphertextMatrix", [(1, "num_rows", F.TYPE_UINT32, one, None), (2, "num_columns", F.TYPE_UINT32, one, None),
                                       (3, "ciphertexts", F.TYPE_MESSAGE, rep, "SerializedCiphertext"),
                                       (4, "packing", F.TYPE_MESSAGE, one, "MatrixPacking")])
    msg("EvaluationKeyMetadata", [(1, "timestamp", F.TYPE_UINT64, one, None), (2, "identifier", F.TYPE_BYTES, one, None)])
    msg("EvaluationKey", [(1, "metadata", F.TYPE_MESSAGE, one, "EvaluationKeyMetadata"),
                          (2, "evaluation_key", F.TYPE_BYTES, one, None)])  # a SerializedEvaluationKey, kept as bytes
    req = msg("PNNSRequest", [(1, "shard_indices", F.TYPE_UINT32, rep, None),
                              (2, "query", F.TYPE_MESSAGE, rep, "SerializedCiphertextMatrix"),
                              (3, "evaluation_key_metadata", F.TYPE_MESSAGE, one, "EvaluationKeyMetadata"),
                              (4, "config_id", F.TYPE_BYTES, one, None),
                              (5, "evaluation_key", F.TYPE_MESSAGE, one, "EvaluationKey"),
                              (6, "shard_ids", F.TYPE_STRING, rep, None)])
    req.oneof_decl.add(name="_evaluation_key")  # proto3 `optional EvaluationKey evaluation_key`
    req.field[4].proto3_optional = True
    req.field[4].oneof_index = 0
    msg("PNNSShardResponse", [(1, "reply", F.TYPE_MESSAGE, rep, "SerializedCiphertextMatrix"),
                              (2, "entry_ids", F.TYPE_UINT64, rep, None), (3, "entry_metadatas", F.TYPE_BYTES, rep, None)])
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    return {n: message_factory.GetMessageClass(pool.FindMessageTypeByName("t." + n))
            for n in ["PNNSRequest", "PNNSShardResponse", "SerializedCiphertextMatrix"]}


def test_protobuf_parses_the_restatement():
    P = protobuf_classes()
    r = P["PNNSRequest"].FromString(KAT_REQUEST_KEY)
    assert list(r.shard_indices) == [3, 7] and r.config_id == b"\x09" and list(r.shard_ids) == ["z"]
    assert (r.evaluation_key.metadata.timestamp, r.evaluation_key.metadata.identifier) == (5, b"k0")
    assert r.evaluation_key.evaluation_key == KEY
    m = r.query[0]
    assert (m.num_rows, m.num_columns, m.packing.WhichOneof("matrix_packing_type")) == (1, 2, "dense_row")
    assert m.ciphertexts[0].seeded.poly0 == POLY0 and m.ciphertexts[0].seeded.seed == SEED
    s = P["PNNSShardResponse"].FromString(KAT_RESPONSE_2)
    assert list(s.entry_ids) == [7, 8, 9] and list(s.entry_metadatas) == [b"\xaa", b"", b"\xbb\xcc"]
    assert len(s.reply) == 2 and s.reply[1].packing.WhichOneof("matrix_packing_type") == "dense_column"
    full = s.reply[0].ciphertexts[0].full
    assert (full.polys, list(full.skip_lsbs), full.correction_factor) == (b"\x02\x00" + P0 + P1, [1, 2], 1)


def test_protobuf_writes_the_restatements_bytes():
    P = protobuf_classes()
    rng = random.Random(2)
    cts = [("seeded", bytes(rng.randrange(256) for _ in range(22)), bytes(rng.randrange(256) for _ in range(32)))
           for _ in range(3)]
    r = P["PNNSRequest"](shard_indices=[1, 300], config_id=b"cfg", shard_ids=["a", "bc"])
    for _ in range(2):
        m = r.query.add(num_rows=5, num_columns=17)
        m.packing.dense_row.SetInParent()
        for _, p, s in cts:
            c = m.ciphertexts.add()
            c.seeded.poly0, c.seeded.seed = p, s
    r.evaluation_key.metadata.timestamp = 9
    r.evaluation_key.evaluation_key = KEY
    matrix = ref.encode_matrix(5, 17, cts, ref.DENSE_ROW)
    assert r.SerializeToString() == ref.encode_pnns_request([matrix, matrix], [1, 300], None, b"cfg", KEY, (9, b""),
                                                            ["a", "bc"])
    for metadata in ([], [b""], [b"x", b"", b"yz"]):
        s = P["PNNSShardResponse"](entry_ids=[0, 1, 1 << 40], entry_metadatas=metadata)
        for k in range(2):
            m = s.reply.add(num_rows=100000, num_columns=3)
            m.packing.dense_column.SetInParent()
            for i in range(2):
                full = m.ciphertexts.add().full
                full.polys = b"\x02\x00" + bytes([k, i]) * 7
                full.skip_lsbs.extend([k + 1, 0])
                full.correction_factor = 1
        matrices = [([(bytes([k, i]) * 4, bytes([k, i]) * 3) for i in range(2)], [k + 1, 0]) for k in range(2)]
        assert s.SerializeToString() == ref.encode_shard_response(matrices, 100000, 3, [0, 1, 1 << 40], metadata)


# ---- the library's walk, template and plan on the CPU -------------------------------------------------------------------

@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    binary = str(tmp_path_factory.mktemp("emu") / "pnns_proto_emulate")
    subprocess.check_call([NVCC, "-O1", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", binary, EMU_SRC])

    def run(args, data=b""):
        out = subprocess.run([binary] + [str(a) for a in args], input=(data.hex() or ".") + "\n", capture_output=True,
                             text=True, check=True)
        return out.stdout.split("\n")[:-1]

    return run


def emu_query(emu, data, contexts=1, columns=2):
    lines = emu(["query", N, contexts, columns] + BITS, data)
    if lines[0].startswith("error"):
        return ("error", int(lines[0].split()[1]), lines[0].split(" ", 2)[2])
    matrices, cts = [], None
    for line in lines[1:]:
        kind, *at = line.split()
        at = [int(x) for x in at]
        if kind == "matrix":
            cts = []
            matrices.append(cts)
        elif kind == "seeded":
            cts.append(("seeded", data[at[0]:at[0] + SIZES(0)], data[at[1]:at[1] + 32]))
        else:
            cts.append(("full", data[at[0] - 2:at[1] + SIZES(at[3])], at[2:], 1))
    return int(lines[0].split()[1]), matrices


def test_emulated_request_walk(emu):
    assert emu_query(emu, KAT_REQUEST_1) == (1, [[SEEDED]])
    assert emu_query(emu, KAT_REQUEST_2, contexts=2) == (1, [[SEEDED], [SEEDED]])
    lines = emu(["request"], KAT_REQUEST_KEY)
    assert lines[0] == "ok"
    f = [int(x) for x in lines[1].split()]
    want = ref.parse_pnns_request(KAT_REQUEST_KEY)
    assert f[:6] == [1, 1, 1, 1, 2, 1]
    assert KAT_REQUEST_KEY[f[6]:f[6] + f[7]] == want["configId"]
    assert (f[8], f[8] + f[9]) == want["evaluationKey"]
    assert f[10] == 5 and KAT_REQUEST_KEY[f[11]:f[11] + f[12]] == b"k0"
    assert lines[2] == "indices 3 7"
    offset, length = (int(x) for x in lines[3].split()[1].split(":"))
    assert KAT_REQUEST_KEY[offset:offset + length] == b"z"
    # evaluation_key_metadata wins over the metadata inside evaluation_key
    outer = ref.encode_pnns_request([bytes.fromhex(MATRIX_HEX)], metadata=(8, b"o"), evaluation_key=KEY, key_metadata=(5, b"i"))
    f = [int(x) for x in emu(["request"], outer)[1].split()]
    assert f[10] == 8 and outer[f[11]:f[11] + f[12]] == b"o"


def test_emulated_walk_of_random_requests(emu):
    rng = random.Random(3)
    for trial in range(20):
        contexts, rows = rng.randrange(1, 4), rng.randrange(1, 9)
        columns = rng.choice([1, 2, 3, 4])
        count = -(-rows // (2 * (8 // (1 << (columns - 1).bit_length()))))
        matrices, encoded = [], []
        for _ in range(contexts):
            cts = []
            for _ in range(count):
                if rng.random() < 0.3:
                    skips = rng.choice([[], [0, 0], [1, 3]])
                    s = skips or [0, 0]
                    cts.append(("full", pref.full_polys(*(bytes(rng.randrange(256) for _ in range(SIZES(k))) for k in s)),
                                skips, 1))
                else:
                    cts.append(("seeded", bytes(rng.randrange(256) for _ in range(22)),
                                bytes(rng.randrange(256) for _ in range(32))))
            matrices.append([ct if ct[0] == "seeded" else (ct[0], ct[1], list(ct[2]) or [0, 0], 1) for ct in cts])
            encoded.append(ref.encode_matrix(rows, columns, cts, ref.DENSE_ROW))
        data = ref.encode_pnns_request(encoded, shard_indices=[trial], config_id=b"c" * trial)
        assert emu_query(emu, data, contexts, columns) == (rows, matrices), trial


REFUSALS = {
    "wrongCiphertextMatrixCount": (lambda m: ref.encode_pnns_request([m]), 2, 2),
    "wrongMatrixPacking(got: .diagonal": (lambda m: ref.encode_pnns_request(
        [ref.encode_matrix(1, 2, [SEEDED], ref.DIAGONAL)]), 1, 2),
    "wrongMatrixPacking(got: .denseColumn": (lambda m: ref.encode_pnns_request(
        [ref.encode_matrix(1, 2, [SEEDED], ref.DENSE_COLUMN)]), 1, 2),
    "unsetOneof(MatrixPacking": (lambda m: ref.encode_pnns_request([ref.encode_matrix(1, 2, [SEEDED], None)]), 1, 2),
    "invalidMatrixDimensions(rowCount: 1, columnCount: 2)": (lambda m: ref.encode_pnns_request([m]), 1, 3),
    "invalidMatrixDimensions(rowCount: 0": (lambda m: ref.encode_pnns_request(
        [ref.encode_matrix(0, 2, [SEEDED], ref.DENSE_ROW)]), 1, 2),
    "wrongCiphertextCount(got: 2, expected: 1)": (lambda m: ref.encode_pnns_request(
        [ref.encode_matrix(1, 2, [SEEDED, SEEDED], ref.DENSE_ROW)]), 1, 2),
    "invalidMatrixDimensions: query matrices of 1 and 2 rows": (lambda m: ref.encode_pnns_request(
        [m, ref.encode_matrix(2, 2, [SEEDED], ref.DENSE_ROW)]), 2, 2),
    "invalid seed": (lambda m: ref.encode_pnns_request(
        [ref.encode_matrix(1, 2, [("seeded", POLY0, SEED[:31])], ref.DENSE_ROW)]), 1, 2),
    "serializedBufferSizeMismatch(poly0": (lambda m: ref.encode_pnns_request(
        [ref.encode_matrix(1, 2, [("seeded", POLY0[:-1], SEED)], ref.DENSE_ROW)]), 1, 2),
    "truncated": (lambda m: KAT_REQUEST_1[:-1], 1, 2),
    "a singular message given twice": (lambda m: ref.encode_pnns_request([m]) + bytes.fromhex("2a00" "2a00"), 1, 2),
}


@pytest.mark.parametrize("case", list(REFUSALS))
def test_emulated_refusals(emu, case):
    make, contexts, columns = REFUSALS[case]
    got = emu_query(emu, make(bytes.fromhex(MATRIX_HEX)), contexts, columns)
    assert got[:2] == ("error", ERR_INVALID), got
    assert case in got[2], got


@pytest.mark.parametrize("metadata", [[], [b""], [b"\xaa", b"", b"\xbb\xcc"]])
@pytest.mark.parametrize("contexts", [1, 2, 3])
def test_emulated_response_template(emu, contexts, metadata):
    rng = random.Random(contexts * 10 + len(metadata))
    replies, rows, columns = 3, 100000, 2
    sizes = [(8, 6, 1, 2), (9, 5, 0, 3), (10, 10, 0, 0)][:contexts]
    matrices, polys = [], b""
    for b0, b1, s0, s1 in sizes:
        rs = [(bytes(rng.randrange(256) for _ in range(b0)), bytes(rng.randrange(256) for _ in range(b1)))
              for _ in range(replies)]
        matrices.append((rs, [s0, s1]))
        polys += b"".join(p0 + p1 for p0, p1 in rs)
    ids = [7, 300, 1 << 33]
    args = ["response", replies, rows, columns, ",".join(map(str, ids)),
            ",".join(m.hex() or "~" for m in metadata) if metadata else "-", contexts]
    for size in sizes:
        args += list(size)
    framed = bytes.fromhex(emu(args, polys)[0])
    assert framed == ref.encode_shard_response(matrices, rows, columns, ids, metadata)
    if sizes[0][:2] == sizes[-1][:2]:  # one reply size: the library's read walk over one-row polys of 8 + 6 bytes
        lines = emu(["read", N, 5, contexts], framed)
        assert lines[0] == f"ok {rows} {columns} {replies}"
        for k, line in enumerate(lines[1:1 + contexts]):
            _, s0, s1, *at = line.split()
            assert [int(s0), int(s1)] == matrices[k][1]
            assert [framed[int(a):int(a) + 14] for a in at] == [p0 + p1 for p0, p1 in matrices[k][0]]
        assert lines[1 + contexts] == "ids " + " ".join(map(str, ids))


def test_emulated_read_refusals(emu):
    assert emu(["read", N, 5, 2], KAT_RESPONSE_1)[0].startswith(f"error {ERR_INVALID} wrongCiphertextMatrixCount")
    row = bytes.fromhex("0a24" "0803" "1001" "1a1a" + FULL_HEX + "2202" "0a00")  # .denseRow
    assert emu(["read", N, 5, 1], row)[0].startswith(f"error {ERR_INVALID} wrongMatrixPacking")


# ---- the query plan --------------------------------------------------------------------------------------------------

def python_plan(n, rows, columns, db_rows, elements):
    """What PlaintextMatrix._rowDescriptors derives, before the masks are SIMD-encoded."""
    dims = pnns.MatrixDimensions(rows, columns)
    count = pnns.CiphertextMatrix.ciphertextCount(n, dims)
    out = [f"ok {count} {pnns._next_power_of_two(columns)}"]
    if rows > 1:
        for r in range(rows):
            index, mask, rotate = pnns.CiphertextMatrix.denseRowExtraction(n, dims, count, r)
            out.append(f"row {index} {rotate} " + "".join(map(str, mask + [0] * (n - len(mask)))))
    sequence = []
    if (n // 2) // db_rows > 1 and rows > 1:
        try:
            sequence = pnns.GaloisElement.rotationSequence(elements, db_rows, n)
        except Exception as e:  # noqa: BLE001 -- invalidRotationStep
            return ["error", str(e)]
    return out + ["pack" + "".join(f" {s}" for s in sequence)]


def galois_sets(n, db_rows, columns, rows):
    rot = pnns.GaloisElement.rotatingColumns
    config = pnns.MatrixMultiplication.evaluationKeyConfig(pnns.MatrixDimensions(db_rows, columns), rows, n).galoisElements
    sets = [config]
    steps = [s for s in (1, 2, 3, 5, 16) if s < n // 2]
    sets.append([rot(s, n) for s in steps[:2]] + [n * 2 - 1])  # steps 1 and 2 only: multi-step plans
    sets.append([rot(-s, n) for s in steps[:3]])  # only leftward steps: planned by their complements
    return sets


@pytest.mark.parametrize("n", [32, 64])
def test_emulated_plan_matches_row_descriptors(emu, n):
    rng = random.Random(n)
    half = n // 2
    cases = set()
    for rows in list(range(1, 17)) + [31, 32, 33, 64]:
        for columns in sorted({1, 3, 5, 8, half // 2 + 1, half - 1, half}):
            db_rows = rng.choice([1, 3, 5, half // 4, half // 2 - 1, half, half + 3, 3 * n])
            cases.add((rows, columns, max(1, db_rows)))
    checked = 0
    for rows, columns, db_rows in sorted(cases):
        for elements in galois_sets(n, db_rows, columns, rows):
            got = emu(["plan", n, rows, columns, db_rows] + list(elements))
            want = python_plan(n, rows, columns, db_rows, elements)
            if want[0] == "error":
                assert got[0].startswith("error invalidRotationStep"), (rows, columns, db_rows, elements, got)
            else:
                assert got == want, (rows, columns, db_rows, elements)
            checked += 1
    assert checked > 300
