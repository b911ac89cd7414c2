"""PNNS in the reference's protobuf messages at the C5 shape (N = 8192, four 55-bit moduli, 100 000 x 512 database,
one-vector clients): the protobuf call (Server.computeResponsesProto: PNNSRequest in, PNNSShardResponse out, the query
plan derived in the library, keys read in place on every context) against the host composition it replaces (walk each
request and copy its poly0 and seeds per plaintext modulus, EvaluationKey.forContext copies, _clients_wire once per
plaintext modulus, host framing), for 1, 16 and 64 clients, with one plaintext modulus and with one extra 17-bit one.

Rounds of the two paths alternate; each reports its best round.  Prints one JSON line per measurement, then the card
name and power limit read in the same run.
    python tools/bench_pnns_proto.py [--reps 5] [--samples 3]"""
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
import pir_proto_ref as pref  # noqa: E402
import pnns_proto_ref as ref  # noqa: E402
from hecuda import pnns  # noqa: E402

Q8192 = [36028797018652673, 36028797017571329, 36028797017456641, 36028797017276417]
N, ROWS, COLS = 8192, 100000, 512
GROUP = 16  # HECUDA_PNNS_CLIENT_GROUP
EXTRA_T = 114689  # 7 * 2^14 + 1, the 17-bit plaintext modulus of tools/bench_pnns_client.py


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True)
    return out.stdout.strip()


def host_composition(server, messages, keys):
    """The path without the protobuf call.  Returns (responses, host seconds walking and framing)."""
    db = server.database
    sizes = pref.poly_sizes(N, [q.bit_length() for q in Q8192[:db.contexts[0].L]])
    t0 = time.perf_counter()
    per_context = []
    for m in messages:
        ranges = ref.parse_pnns_request(m)["query"]
        per_context.append([ref.parse_matrix(m, b, e, sizes) for b, e in ranges])
    walk = time.perf_counter() - t0
    rows = per_context[0][0][0]
    dims = pnns.MatrixDimensions(rows, COLS)
    replies = []
    for k, matrix in enumerate(db.plaintextMatrices):
        t1 = time.perf_counter()
        poly0 = np.stack([np.frombuffer(b"".join(ct[1] for ct in q[k][3]), np.uint8).reshape(len(q[k][3]), -1)
                          for q in per_context])
        seeds = np.stack([np.frombuffer(b"".join(ct[2] for ct in q[k][3]), np.uint8).reshape(len(q[k][3]), 32)
                          for q in per_context])
        walk += time.perf_counter() - t1
        ks = [key.forContext(matrix.context) for key in keys]
        replies.append(pnns.PnnsWire.computeResponses(matrix, poly0, seeds, dims, ks))
    t2 = time.perf_counter()
    out = []
    for c in range(len(messages)):
        matrices = []
        for k, (r, skips) in enumerate(replies):
            b0 = hecuda.Bfv.serializationByteCount(db.plaintextMatrices[k].context, 1, skips[0])
            matrices.append(([(x[:b0].tobytes(), x[b0:].tobytes()) for x in r[c]], skips))
        out.append(ref.encode_shard_response(matrices, ROWS, rows, db.entryIds, db.entryMetadatas))
    return out, walk + time.perf_counter() - t2


def run(ts, args):
    gs = [hecuda.Context(N, Q8192, t) for t in ts]
    params = pnns.EncryptionParameters(N, ts[0], tuple(Q8192))
    s = pnns.ClientConfig.maxScalingFactor(pnns.COSINE_SIMILARITY, COLS, ts)
    ekc = pnns.MatrixMultiplication.evaluationKeyConfig(pnns.MatrixDimensions(ROWS, COLS), 1, N)
    cc = pnns.ClientConfig(params, s, COLS, ekc, extraPlaintextModuli=ts[1:])
    rng = np.random.default_rng(5)
    vectors = rng.standard_normal((ROWS, COLS)).astype(np.float32)
    db = pnns.Database([pnns.DatabaseRow(i, b"", list(v)) for i, v in enumerate(vectors)])
    processed = pnns.ProcessedDatabase.processOnDevice(db, pnns.ServerConfig(cc), gs)
    client, server = pnns.Client(cc, gs), pnns.Server(processed)
    keys, messages = [], []
    for j in range(64):
        sk = client.generateSecretKey()
        keys.append(client.generateEvaluationKey(sk))
        messages.append(client.requestMessage(vectors[j:j + 1], sk))
    for clients in (1, 16, 64):
        msgs, ks = messages[:clients], keys[:clients]
        got = server.computeResponsesProto(msgs, ks)  # warm-up
        want, _ = host_composition(server, msgs, ks)
        sampled = sorted({0, clients // 2, clients - 1})[:args.samples]
        parity = all(got[c] == want[c] for c in sampled)
        before = hecuda.kernel_launch_count()
        server.computeResponsesProto(msgs, ks)
        launches = hecuda.kernel_launch_count() - before
        groups = -(-clients // GROUP)
        proto, host, frame = [], [], []
        for _ in range(args.reps):  # alternated rounds
            t0 = time.perf_counter()
            server.computeResponsesProto(msgs, ks)
            proto.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            _, f = host_composition(server, msgs, ks)
            host.append(time.perf_counter() - t0)
            frame.append(f)
        tail = len(ref.encode_shard_response([], ROWS, 1, processed.entryIds, processed.entryMetadatas))
        key_bytes = 0
        if len(gs) > 1:  # one forContext copy per extra context: L x 2 x (L + 1) x N words per Galois key
            L = gs[0].L
            key_bytes = (len(gs) - 1) * len(ekc.galoisElements) * L * 2 * (L + 1) * N * 8
        print(json.dumps({
            "plaintext_moduli": len(ts), "clients": clients, "proto_clients_per_s": clients / min(proto),
            "host_composition_clients_per_s": clients / min(host), "host_walk_and_frame_s": min(frame),
            "pcie_in_bytes_per_client": len(msgs[0]), "pcie_out_bytes_per_client": len(got[0]),
            "pcie_out_ids_and_metadata_bytes_per_client": tail, "kernel_launches_per_group": launches / groups,
            "key_copy_bytes_per_client_saved": key_bytes, "sampled_byte_parity": parity}))
    for k in keys:
        k.close()
    processed.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--samples", type=int, default=3)
    args = ap.parse_args()
    run([65537], args)
    run([65537, EXTRA_T], args)
    print(json.dumps({"card": card()}))


if __name__ == "__main__":
    main()
