"""PIR requests and responses in the reference's protobuf messages, on the CPU.

- Known-answer byte strings, written out by hand at N = 16, pin the restatement (tests/pir_proto_ref.py) for
  EncryptedIndices, SerializedEvaluationKey, PIRRequest and PIRResponse.
- A cross-check against google.protobuf, with descriptors built here from the .proto field tables: it parses the
  restatement's bytes to the same values, and messages it builds serialize to the restatement's bytes.  This stands in
  for bytes written by SwiftProtobuf, which cannot be produced here; both follow the same proto3 encoding rules.
- tests/emu/pir_proto_emulate.cu runs the library's own walks, offset tables and response template (pir_proto.hpp,
  protobuf.hpp) on the CPU and must reproduce the restatement, including every refusal."""
import os
import random
import shutil
import subprocess

import pytest

import pir_proto_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_SRC = os.path.join(ROOT, "tests", "emu", "pir_proto_emulate.cu")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ERR_INVALID, ERR_UNSUPPORTED = -1, -2

# N = 16 over rows of 5 and 6 bits: a poly0 is 10 + 12 = 22 bytes; a reply row of 5 bits with skip_lsbs [1, 2] is 8 + 6
N, BITS, REPLY_BITS = 16, [5, 6], [5]
SIZES, REPLY_SIZES = ref.poly_sizes(N, BITS), ref.poly_sizes(N, REPLY_BITS)
POLY0, SEED = bytes(range(22)), bytes(range(32, 64))
SEEDED = ("seeded", POLY0, SEED)
SEEDED_HEX = "0a3c" "0a3a" "0a16" + POLY0.hex() + "1220" + SEED.hex()  # SerializedCiphertext { seeded { poly0 seed } }
KAT_QUERY = bytes.fromhex(SEEDED_HEX + "1001")
KSK_HEX = "0a3e" + SEEDED_HEX  # SerializedKeySwitchKey { key_switch_key { ciphertexts } }
KAT_KEY = bytes.fromhex("0a46" "0a44" "0803" "1240" + KSK_HEX + "1242" "0a40" + KSK_HEX)
P0, P1 = bytes(range(100, 108)), bytes(range(200, 206))
KAT_RESPONSE = bytes.fromhex("0a1c" "0a1a" "1218" "0a10" "0200" + P0.hex() + P1.hex() + "12020102" "1801")
KAT_REQUEST = bytes.fromhex("0802" "1240" + KAT_QUERY.hex() + "1a06" "0805" "12026162" "220109" "2a0173"
                            "328f01" "128c01" + KAT_KEY.hex())


def test_known_answers():
    assert ref.encode_encrypted_indices([SEEDED], 1) == KAT_QUERY
    assert ref.parse_encrypted_indices(KAT_QUERY, SIZES) == ([SEEDED], 1)
    assert ref.encode_evaluation_key([(3, [SEEDED])], [SEEDED]) == KAT_KEY
    assert ref.parse_evaluation_key(KAT_KEY, SIZES, 1) == ({3: [SEEDED]}, [SEEDED])
    assert ref.encode_pir_response([[(P0, P1)]], [1, 2]) == KAT_RESPONSE
    assert ref.parse_pir_response(KAT_RESPONSE, REPLY_SIZES) == [[("full", b"\x02\x00" + P0 + P1, [1, 2], 1)]]
    request = ref.encode_pir_request(2, KAT_QUERY, (5, b"ab"), b"\x09", "s", KAT_KEY)
    assert request == KAT_REQUEST
    fields = ref.parse_pir_request(KAT_REQUEST)
    assert (fields["shardIndex"], fields["shardId"], fields["configurationHash"]) == (2, "s", b"\x09")
    assert (fields["keyTimestamp"], fields["keyIdentifier"]) == (5, b"ab")
    assert KAT_REQUEST[fields["query"][0]:sum(fields["query"])] == KAT_QUERY
    assert KAT_REQUEST[fields["evaluationKey"][0]:sum(fields["evaluationKey"])] == KAT_KEY


# ---- google.protobuf -------------------------------------------------------------------------------------------------

def protobuf_classes():
    pytest.importorskip("google.protobuf")
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    F = descriptor_pb2.FieldDescriptorProto
    fd = descriptor_pb2.FileDescriptorProto(name="pir_proto_test.proto", package="t", syntax="proto3")
    one, rep = F.LABEL_OPTIONAL, F.LABEL_REPEATED

    def msg(name, fields, oneof=None, parent=None):
        m = (parent.nested_type if parent else fd.message_type).add(name=name)
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
                                 (2, "full", F.TYPE_MESSAGE, one, "SerializedFullCiphertext")], oneof="serialized_ciphertext_type")
    msg("SerializedCiphertextVec", [(1, "ciphertexts", F.TYPE_MESSAGE, rep, "SerializedCiphertext")])
    msg("SerializedKeySwitchKey", [(1, "key_switch_key", F.TYPE_MESSAGE, one, "SerializedCiphertextVec")])
    galois = msg("SerializedGaloisKey", [(1, "key_switch_keys", F.TYPE_MESSAGE, rep, "SerializedGaloisKey.KeySwitchKeysEntry")])
    entry = msg("KeySwitchKeysEntry", [(1, "key", F.TYPE_UINT64, one, None),
                                       (2, "value", F.TYPE_MESSAGE, one, "SerializedKeySwitchKey")], parent=galois)
    entry.options.map_entry = True
    msg("SerializedRelinKey", [(1, "relin_key", F.TYPE_MESSAGE, one, "SerializedKeySwitchKey")])
    msg("SerializedEvaluationKey", [(1, "galois_key", F.TYPE_MESSAGE, one, "SerializedGaloisKey"),
                                    (2, "relin_key", F.TYPE_MESSAGE, one, "SerializedRelinKey")])
    msg("EncryptedIndices", [(1, "ciphertexts", F.TYPE_MESSAGE, rep, "SerializedCiphertext"),
                             (2, "num_pir_calls", F.TYPE_UINT64, one, None)])
    msg("EvaluationKeyMetadata", [(1, "timestamp", F.TYPE_UINT64, one, None), (2, "identifier", F.TYPE_BYTES, one, None)])
    msg("EvaluationKey", [(1, "metadata", F.TYPE_MESSAGE, one, "EvaluationKeyMetadata"),
                          (2, "evaluation_key", F.TYPE_MESSAGE, one, "SerializedEvaluationKey")])
    req = msg("PIRRequest", [(1, "shard_index", F.TYPE_UINT32, one, None), (2, "query", F.TYPE_MESSAGE, one, "EncryptedIndices"),
                             (3, "evaluation_key_metadata", F.TYPE_MESSAGE, one, "EvaluationKeyMetadata"),
                             (4, "configuration_hash", F.TYPE_BYTES, one, None), (5, "shard_id", F.TYPE_STRING, one, None),
                             (6, "evaluation_key", F.TYPE_MESSAGE, one, "EvaluationKey")])
    req.oneof_decl.add(name="_shard_id")  # proto3 `optional string shard_id`
    req.field[4].proto3_optional = True
    req.field[4].oneof_index = 0
    msg("PIRResponse", [(1, "replies", F.TYPE_MESSAGE, rep, "SerializedCiphertextVec")])
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    names = ["SerializedCiphertext", "SerializedEvaluationKey", "EncryptedIndices", "PIRRequest", "PIRResponse",
             "SerializedKeySwitchKey"]
    return {n: message_factory.GetMessageClass(pool.FindMessageTypeByName("t." + n)) for n in names}


def test_protobuf_parses_the_restatement():
    P = protobuf_classes()
    q = P["EncryptedIndices"].FromString(KAT_QUERY)
    assert q.num_pir_calls == 1 and q.ciphertexts[0].seeded.poly0 == POLY0 and q.ciphertexts[0].seeded.seed == SEED
    k = P["SerializedEvaluationKey"].FromString(KAT_KEY)
    assert list(k.galois_key.key_switch_keys) == [3]
    assert k.galois_key.key_switch_keys[3].key_switch_key.ciphertexts[0].seeded.poly0 == POLY0
    assert k.relin_key.relin_key.key_switch_key.ciphertexts[0].seeded.seed == SEED
    r = P["PIRResponse"].FromString(KAT_RESPONSE)
    full = r.replies[0].ciphertexts[0].full
    assert (full.polys, list(full.skip_lsbs), full.correction_factor) == (b"\x02\x00" + P0 + P1, [1, 2], 1)
    req = P["PIRRequest"].FromString(KAT_REQUEST)
    assert (req.shard_index, req.shard_id, req.configuration_hash) == (2, "s", b"\x09")
    assert req.evaluation_key_metadata.timestamp == 5 and req.query.SerializeToString() == KAT_QUERY
    assert req.evaluation_key.evaluation_key.SerializeToString() == KAT_KEY


def test_protobuf_writes_the_restatements_bytes():
    P = protobuf_classes()
    rng = random.Random(1)
    cts = [("seeded", bytes(rng.randrange(256) for _ in range(22)), bytes(rng.randrange(256) for _ in range(32)))
           for _ in range(3)]
    q = P["EncryptedIndices"](num_pir_calls=2)
    for _, p, s in cts:
        c = q.ciphertexts.add()
        c.seeded.poly0, c.seeded.seed = p, s
    assert q.SerializeToString() == ref.encode_encrypted_indices(cts, 2)
    k = P["SerializedEvaluationKey"]()
    for _, p, s in cts[:2]:
        c = k.galois_key.key_switch_keys[9].key_switch_key.ciphertexts.add()
        c.seeded.poly0, c.seeded.seed = p, s
    relin = k.relin_key.relin_key.key_switch_key.ciphertexts.add()
    relin.seeded.poly0, relin.seeded.seed = cts[2][1], cts[2][2]
    assert k.SerializeToString(deterministic=True) == ref.encode_evaluation_key([(9, cts[:2])], cts[2:])
    r = P["PIRResponse"]()
    for reply in range(2):
        vec = r.replies.add()
        for chunk in range(3):
            full = vec.ciphertexts.add().full
            full.polys = b"\x02\x00" + bytes([reply, chunk]) * 7
            full.skip_lsbs.extend([1, 2])
            full.correction_factor = 1
    assert r.SerializeToString() == ref.encode_pir_response(
        [[(bytes([reply, chunk]) * 4, bytes([reply, chunk]) * 3) for chunk in range(3)] for reply in range(2)], [1, 2])
    req = P["PIRRequest"](shard_index=7, configuration_hash=b"h", shard_id="")
    req.query.CopyFrom(q)
    req.evaluation_key.metadata.timestamp = 3
    req.evaluation_key.evaluation_key.CopyFrom(k)
    assert req.SerializeToString(deterministic=True) == ref.encode_pir_request(
        7, ref.encode_encrypted_indices(cts, 2), None, b"h", "", ref.encode_evaluation_key([(9, cts[:2])], cts[2:]),
        key_metadata=(3, b""))


def test_map_entry_order_loads_the_same_key():
    P = protobuf_classes()
    keys = [(3, [SEEDED]), (31, [("seeded", POLY0[::-1], SEED[::-1])]), (7, [("seeded", bytes(22), bytes(32))])]
    a, b = ref.encode_evaluation_key(keys), ref.encode_evaluation_key(keys[::-1])
    assert a != b
    assert ref.parse_evaluation_key(a, SIZES, 1) == ref.parse_evaluation_key(b, SIZES, 1)
    assert P["SerializedEvaluationKey"].FromString(a) == P["SerializedEvaluationKey"].FromString(b)


# ---- the library's walk on the CPU -----------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    binary = str(tmp_path_factory.mktemp("emu") / "pir_proto_emulate")
    subprocess.check_call([NVCC, "-O1", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", binary, EMU_SRC])

    def run(args, data, env=None):
        out = subprocess.run([binary] + [str(a) for a in args], input=(data.hex() or ".") + "\n", capture_output=True,
                             text=True, check=True, env=dict(os.environ, **(env or {})))
        return out.stdout.split("\n")[:-1]

    return run


def emu_query(emu, data, expect=None):
    lines = emu(["query", N] + BITS, data, {"EXPECT": expect} if expect else None)
    if lines[0].startswith("error"):
        return ("error", int(lines[0].split()[1]))
    _, calls, count = lines[0].split()
    cts = []
    for line in lines[1:]:
        kind, *at = line.split()
        at = [int(x) for x in at]
        if kind == "seeded":
            cts.append(("seeded", data[at[0]:at[0] + SIZES(0)], data[at[1]:at[1] + 32]))
        else:
            start = at[0] - 2
            end = at[1] + SIZES(at[3])
            cts.append(("full", data[start:end], at[2:], 1))
    assert len(cts) == int(count)
    return cts, int(calls)


def random_query(rng, count, full_every=0):
    cts = []
    for i in range(count):
        if full_every and i % full_every == 0:
            skips = rng.choice([[], [0, 0], [1, 3]])
            s = skips or [0, 0]
            cts.append(("full", ref.full_polys(*(bytes(rng.randrange(256) for _ in range(SIZES(k))) for k in s)),
                        skips, 1))
        else:
            cts.append(("seeded", bytes(rng.randrange(256) for _ in range(22)), bytes(rng.randrange(256) for _ in range(32))))
    return cts


def normalized(cts):
    return [ct if ct[0] == "seeded" else (ct[0], ct[1], list(ct[2]) or [0, 0], ct[3]) for ct in cts]


def test_emulated_query_walk(emu):
    assert emu_query(emu, KAT_QUERY) == ([SEEDED], 1)
    rng = random.Random(2)
    for count, full_every in [(1, 0), (5, 2), (4, 1)]:
        cts = random_query(rng, count, full_every)
        data = ref.encode_encrypted_indices(cts, 3)
        assert ref.parse_encrypted_indices(data, SIZES) == (normalized(cts), 3)
        assert emu_query(emu, data) == (normalized(cts), 3)
        assert emu_query(emu, data, f"3 {count}") == (normalized(cts), 3)


def emu_key(emu, data, count=1):
    lines = emu(["key", N, count] + BITS, data)
    if lines[0].startswith("error"):
        return ("error", int(lines[0].split()[1]))

    def cts(parts):
        return [("seeded", data[int(p):int(p) + SIZES(0)], data[int(s):int(s) + 32]) for p, s in
                (x.split(":") for x in parts)]

    relin, galois = None, {}
    for line in lines[1:]:
        kind, *rest = line.split()
        if kind == "relin":
            relin = cts(rest)
        else:
            galois[int(rest[0])] = cts(rest[1:])
    return galois, relin


def test_emulated_key_walk(emu):
    assert emu_key(emu, KAT_KEY) == ref.parse_evaluation_key(KAT_KEY, SIZES, 1)
    rng = random.Random(3)
    keys = [(e, random_query(rng, 2)) for e in (3, 7, 31, 1 << 40)]
    for order in (keys, keys[::-1]):
        for relin in (None, random_query(rng, 2)):
            data = ref.encode_evaluation_key(order, relin)
            want = ref.parse_evaluation_key(data, SIZES, 2)
            assert emu_key(emu, data, 2) == want
            assert list(want[0]) == [e for e, _ in order]


def test_emulated_request_walk(emu):
    lines = emu(["request"], KAT_REQUEST)
    f = ref.parse_pir_request(KAT_REQUEST)
    shard = KAT_REQUEST.index(b"\x2a\x01s") + 2
    assert lines == ["ok", "shard_index 2", f"shard_id 1 {shard} 1",
                     f"configuration_hash {KAT_REQUEST.index(b'\x22\x01\x09') + 2} 1",
                     f"query 1 {f['query'][0]} {f['query'][1]}",
                     f"evaluation_key 1 {f['evaluationKey'][0]} {f['evaluationKey'][1]}",
                     f"key_metadata 1 5 {KAT_REQUEST.index(b'ab')} 2"]
    # the metadata inside evaluation_key stands in for an absent evaluation_key_metadata
    inner = ref.encode_pir_request(evaluation_key=KAT_KEY, key_metadata=(9, b"xyz"))
    lines = emu(["request"], inner)
    assert lines[-1] == f"key_metadata 1 9 {inner.index(b'xyz')} 3"
    assert ref.parse_pir_request(inner)["keyTimestamp"] == 9


def test_emulated_response_template(emu):
    rng = random.Random(4)
    for indices, chunks, skips in [(1, 1, [1, 2]), (2, 3, [0, 4]), (3, 2, [2, 2])]:
        b0, b1 = REPLY_SIZES(skips[0]), REPLY_SIZES(skips[1])
        polys = [[(bytes(rng.randrange(256) for _ in range(b0)), bytes(rng.randrange(256) for _ in range(b1)))
                  for _ in range(chunks)] for _ in range(indices)]
        flat = b"".join(p0 + p1 for reply in polys for p0, p1 in reply)
        framed = bytes.fromhex(emu(["response", indices, chunks, b0, b1] + skips, flat)[0])
        assert framed == ref.encode_pir_response(polys, skips)
        lines = emu(["read", N, REPLY_BITS[0], indices, chunks] + skips, framed)
        offsets = [int(x) for x in lines[0].split()[1:]]
        assert [framed[o:o + b0] for o in offsets] == [p0 for reply in polys for p0, _ in reply]
    assert emu(["read", N, 5, 2, 1, 1, 2], KAT_RESPONSE)[0].startswith(f"error {ERR_INVALID}")


def refusals():
    """(name, message, expected code, $EXPECT) for the query walk"""
    ok = ref.encode_encrypted_indices([SEEDED], 1)
    seeded_body = bytes.fromhex("0a16") + POLY0 + bytes.fromhex("1220") + SEED
    return [
        ("truncated length", ok[:-3], ERR_INVALID, None),
        ("varint over 10 bytes", ok + b"\x10" + b"\xff" * 10 + b"\x01", ERR_INVALID, None),
        ("group", ok + b"\x1b\x1c", ERR_INVALID, None),
        ("wrong wire type", b"\x0d\x00\x00\x00\x00" + ok, ERR_INVALID, None),
        ("duplicate singular field",
         ref.field_bytes(1, ref.field_bytes(1, seeded_body) + ref.field_bytes(1, seeded_body)) + b"\x10\x01", ERR_INVALID, None),
        ("unset oneof", ref.field_bytes(1, b"") + b"\x10\x01", ERR_INVALID, None),
        ("31-byte seed", ref.encode_encrypted_indices([("seeded", POLY0, SEED[:31])], 1), ERR_INVALID, None),
        ("wrong poly0 size", ref.encode_encrypted_indices([("seeded", POLY0 + b"\0", SEED)], 1), ERR_INVALID, None),
        ("num_pir_calls", ok, ERR_INVALID, "2 1"),
        ("ciphertext count", ok, ERR_INVALID, "1 2"),
        ("correction factor", ref.encode_encrypted_indices([("full", ref.full_polys(POLY0, POLY0), [], 2)], 1),
         ERR_UNSUPPORTED, None),
        ("correction factor unset", ref.encode_encrypted_indices([("full", ref.full_polys(POLY0, POLY0), [], 0)], 1),
         ERR_UNSUPPORTED, None),
        ("full polys size", ref.encode_encrypted_indices([("full", ref.full_polys(POLY0, POLY0[1:]), [], 1)], 1),
         ERR_INVALID, None),
    ]


@pytest.mark.parametrize("case", [r[0] for r in refusals()])
def test_emulated_query_refusals(emu, case):
    _, data, code, expect = next(r for r in refusals() if r[0] == case)
    assert emu_query(emu, data, expect) == ("error", code)
    if expect is None:  # the restatement refuses the same message
        with pytest.raises(ref.ProtoError) as e:
            ref.parse_encrypted_indices(data, SIZES)
        assert e.value.kind == ("unsupported" if code == ERR_UNSUPPORTED else "invalid")


def test_emulated_key_refusals(emu):
    full = ("full", ref.full_polys(POLY0, POLY0), [], 1)
    cases = {
        "duplicate element": (ref.encode_evaluation_key([(3, [SEEDED]), (3, [SEEDED])]), ERR_INVALID),
        "full key ciphertexts": (ref.encode_evaluation_key([(3, [full])]), ERR_UNSUPPORTED),
        "ciphertext count": (ref.encode_evaluation_key([(3, [SEEDED, SEEDED])]), ERR_INVALID),
        "duplicate galois_key": (KAT_KEY[:72] + KAT_KEY, ERR_INVALID),
    }
    for name, (data, code) in cases.items():
        assert emu_key(emu, data) == ("error", code), name
        with pytest.raises(ref.ProtoError):
            ref.parse_evaluation_key(data, SIZES, 1)
