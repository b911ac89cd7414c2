"""PIR in the reference's protobuf messages at the C4 shape (2^20 x 64 B, N = 4096): the protobuf call
(PirWire.computeResponsesProto: EncryptedIndices in, PIRResponse out, walked and framed around the device pipeline)
against the host composition it replaces (walk each message and copy its poly0 and seeds into contiguous arrays, call
computeResponses (_clients_wire), frame every reply on the host), for 1, 16 and 64 clients; and the loading of 16 and
64 evaluation keys from SerializedEvaluationKey messages against fromSerializedMany of the same payloads.

Prints one JSON line per measurement, then the card name and power limit read in the same run.
    python tools/bench_pir_proto.py [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "swift-homomorphic-encryption_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402

import hecuda  # noqa: E402
import pir_proto_ref as ref  # noqa: E402
from hecuda import pir  # noqa: E402

PIR_MODULI = [134176769, 268369921, 268361729]  # n_4096_logq_27_28_28_logt_5 (EncryptionParameters.swift:357-367)
N, T = 4096, 17


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True)
    return out.stdout.strip()


def best(fn, reps):
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return min(times)


def host_composition(g, server, messages, keys):
    """The path without the protobuf call: host walk + copy, _clients_wire, host framing.  Returns (responses,
    host seconds spent walking and framing)."""
    t0 = time.perf_counter()
    sz = ref.poly_sizes(N, [q.bit_length() for q in PIR_MODULI[:g.L]])
    parsed = [ref.parse_encrypted_indices(m, sz)[0] for m in messages]
    poly0 = np.frombuffer(b"".join(ct[1] for q in parsed for ct in q), np.uint8).reshape(len(messages), len(parsed[0]), -1)
    seeds = np.frombuffer(b"".join(ct[2] for q in parsed for ct in q), np.uint8).reshape(len(messages), len(parsed[0]), 32)
    walk = time.perf_counter() - t0
    replies, skips = pir.PirWire.computeResponses(server, poly0, seeds, keys)
    t1 = time.perf_counter()
    half = hecuda.Bfv.serializationByteCount(g, 1, skips[0])
    out = [ref.encode_pir_response([[(r[:half].tobytes(), r[half:].tobytes()) for r in reply] for reply in client], skips)
           for client in replies]
    return out, walk + time.perf_counter() - t1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    g = hecuda.Context(N, PIR_MODULI, T)
    param = pir.MulPir.generateParameter(pir.IndexPirConfig(1 << 20, 64, 2, 1, True, "hybridCompression", False), g)
    chunks = -(-param.encodedEntrySize // pir.bytesPerPlaintext(g))
    rows = np.random.default_rng(1).integers(0, T, size=(chunks * int(np.prod(param.dimensions)), N), dtype=np.uint64)
    server = pir.MulPirServer(param, g, [pir.ProcessedDatabase(g, rows, None, evalFormat=False)])
    del rows
    client = pir.MulPirClient(param, g)
    rng = np.random.default_rng(2)
    forms, key_messages, queries = [], [], []
    for _ in range(64):
        sk = hecuda.SecretKey.generate(g)
        key, form = hecuda.EvaluationKey.generate(g, client.evaluationKeyConfig, sk, wire=True)
        key.close()
        forms.append(form)
        key_messages.append(pir.evaluationKeyMessage(g, form))
        queries.append(client.queryMessage([int(rng.integers(param.entryCount))], sk))
    keys = hecuda.EvaluationKey.fromProtoMany(g, key_messages)
    wire_in = sum(len(ct[1]) + len(ct[2]) for ct in ref.parse_encrypted_indices(
        queries[0], ref.poly_sizes(N, [q.bit_length() for q in PIR_MODULI[:g.L]]))[0])
    skips = pir.skipLSBsForDecryption(g)
    wire_out = chunks * sum(hecuda.Bfv.serializationByteCount(g, 1, s) for s in skips)
    for clients in (1, 16, 64):
        msgs, ks = queries[:clients], keys[:clients]
        got = pir.PirWire.computeResponsesProto(server, msgs, ks)  # warm-up (and the graphs / caches of the shape)
        want, _ = host_composition(g, server, msgs, ks)
        assert got == want, "the protobuf call and the host composition differ"
        before = hecuda.kernel_launch_count()
        pir.PirWire.computeResponsesProto(server, msgs, ks)
        launches = hecuda.kernel_launch_count() - before
        groups = -(-clients // 16)
        proto_s = best(lambda: pir.PirWire.computeResponsesProto(server, msgs, ks), args.reps)
        host_s = best(lambda: host_composition(g, server, msgs, ks), args.reps)
        host_frame_s = min(host_composition(g, server, msgs, ks)[1] for _ in range(args.reps))
        print(json.dumps({
            "clients": clients, "proto_clients_per_s": clients / proto_s, "host_composition_clients_per_s": clients / host_s,
            "host_walk_and_frame_s": host_frame_s, "pcie_in_bytes_per_client": {"proto": len(msgs[0]), "wire": wire_in},
            "pcie_out_bytes_per_client": {"proto": len(got[0]), "wire": wire_out},
            "kernel_launches_per_group": launches / groups}))
    for k in keys:
        k.close()
    for count in (16, 64):
        def load_proto():
            for k in hecuda.EvaluationKey.fromProtoMany(g, key_messages[:count]):
                k.close()

        def load_serialized():
            for k in hecuda.EvaluationKey.fromSerializedMany(g, forms[:count]):
                k.close()

        load_proto(), load_serialized()
        print(json.dumps({"keys": count, "fromProtoMany_s": best(load_proto, args.reps),
                          "fromSerializedMany_s": best(load_serialized, args.reps),
                          "key_message_bytes": len(key_messages[0])}))
    print(json.dumps({"card": card()}))
    g.close()


if __name__ == "__main__":
    main()
