"""Sharded SimplePIR restated in plain Python, the checker of hecuda.simple_pir's sharding:

    DatabaseMap.shardDatabase             SimplePir/DatabaseMap.swift:82-110
    ShardMap                              SimplePir/SimplePir+Shards.swift:18-45
    SimplePirClientForAllShards           SimplePir/SimplePir+Shards.swift:47-173, over oracle.simple_pir_oracle.Client

The reference draws each entry's shard permutation from SystemRandomNumberGenerator, so shard_database takes the
permutations as an argument: perms[e] is entry e's shuffled shard order.
"""
from __future__ import annotations

import numpy as np


def shard_database(entries, shard_count: int, chunk_size: int, perms):
    """entries: (originalIndex, bytes) pairs -> (map entries [(originalIndex, size, [(shardIndex, index)])], shards as
    rows x chunk_size uint8 arrays)."""
    shards = [[] for _ in range(shard_count)]
    mapped = []
    for e, (original, value) in enumerate(entries):
        value = bytes(value)
        chunks = []
        for c, start in enumerate(range(0, len(value), chunk_size)):
            piece = value[start:start + chunk_size]
            shard = int(perms[e][c % shard_count])
            chunks.append((shard, len(shards[shard])))
            shards[shard].append(piece + bytes(chunk_size - len(piece)))
        mapped.append((original, len(value), chunks))
    return mapped, [np.frombuffer(b"".join(rows), dtype=np.uint8).reshape(len(rows), chunk_size) for rows in shards]


class ShardMap:
    def __init__(self, mapped):
        self.mapping = {original: (size, chunks) for original, size, chunks in mapped}
        self.shard_count = len({s for _, chunks in self.mapping.values() for s, _ in chunks})
        self.maximum_chunk_count = max((len(chunks) for _, chunks in self.mapping.values()), default=0)
        self.chunks_per_shard = -(-self.maximum_chunk_count // self.shard_count)


class ClientForAllShards:
    """clients: one oracle Client per shard (in shard order)."""

    def __init__(self, mapped, chunk_size: int, clients):
        self.map, self.chunk_size, self.clients = ShardMap(mapped), chunk_size, clients
        assert self.map.shard_count == len(clients)

    def query(self, index: int):
        """-> per shard, chunksPerShard (row index, (query, results)): the entry's chunks first, then index 0."""
        wanted = [[] for _ in self.clients]
        entry = self.map.mapping.get(index)
        if entry is not None:
            for shard, row in entry[1]:
                wanted[shard].append(row)
        for rows in wanted:
            rows += [0] * (self.map.chunks_per_shard - len(rows))
        return [[(row, client.query(row)) for row in rows] for client, rows in zip(self.clients, wanted)]

    def decrypt(self, responses, queries, index: int):
        """responses[s][i] answers queries[s][i] -> the entry's bytes, or None for an index the map does not hold."""
        plain = [[client.decrypt(np.asarray(r, dtype=np.uint64), q[1][1], q[0]) for r, q in zip(rs, qs)]
                 for client, rs, qs in zip(self.clients, responses, queries)]
        entry = self.map.mapping.get(index)
        chunks = entry[1] if entry is not None else []
        out = b""
        for c in range(self.map.maximum_chunk_count):
            shard, row = chunks[c] if c < len(chunks) else (0, 0)
            at = max(i for i, q in enumerate(queries[shard]) if q[0] == row)
            out += plain[shard][at][:self.chunk_size]
        return None if entry is None else out[:entry[0]]
