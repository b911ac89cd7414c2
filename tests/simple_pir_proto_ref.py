"""An independent restatement of the SimplePIR protobuf messages, written from the reference's .proto files
(pir/v1/simple_pir.proto, api/pir/v1/pir.proto) and PirConversion.swift:380-518.  Encoders give SwiftProtobuf's bytes
(fields in number order, proto3 zero scalars omitted, set messages written even when empty, repeated scalars packed,
every element of a repeated message or bytes field written).

    SimplePIRMatrix            1 row_count  2 col_count  3 data (packed uint64, row-major)
    SimplePIRRequest           1 request (SimplePIRMatrix)  2 shard_index  3 configuration_hash
    SimplePIRResponse          1 response (SimplePIRMatrix)
    SimplePIREncryptionParams  1 lattice_dimension  2 error_std_dev (double, fixed64)  3 plaintext_bits  4 ciphertext_bits
    SimplePIRParameters        1 encryption_params  2 a_seed  3 entry_size_in_bytes  4 entries_per_column
                               5 chunks_per_entry  6 database_columns
    DatabaseMapping            1 entries { 1 original_index  2 size  3 chunks { 1 shard_index  2 index } }  2 chunk_size
    SimplePIRConfig            1 database_mapping  2 params  3 hint_identifiers

The b_offset map of the request digit planes is restated from simple_pir.cuh's layout description (8 x 32 tiles,
query-tile-major; lane = query % 8 * 4 + (column % 16) / 4, byte (column / 16 % 2) * 4 + column % 4 of its 8)."""
import struct

from pir_proto_ref import LEN, ProtoError, field_bytes, field_scalar, fields, packed, read_varint, varint

FIXED64 = 1


def encode_matrix(rows, columns, data):
    """Array2d.proto(): data row-major, as uint64."""
    return field_scalar(1, rows) + field_scalar(2, columns) + packed(3, [int(v) for v in data])


def encode_request(rows, columns, data, shard_index=0, configuration_hash=b""):
    return (field_bytes(1, encode_matrix(rows, columns, data)) + field_scalar(2, shard_index) +
            (field_bytes(3, configuration_hash) if configuration_hash else b""))


def encode_response(rows, columns, data):
    return field_bytes(1, encode_matrix(rows, columns, data))


def split_packed(number, values, cuts):
    """`values` as several packed runs, cut before each index in `cuts` (protobuf concatenates them)."""
    bounds = [0] + list(cuts) + [len(values)]
    return b"".join(field_bytes(number, b"".join(varint(int(v)) for v in values[a:b])) for a, b in zip(bounds, bounds[1:]))


def unpacked(number, values):
    return b"".join(field_scalar(number, int(v)) if v else varint(number << 3) + b"\x00" for v in values)


def encode_request_with(rows, columns, data_field, shard_index=0):
    """A request whose matrix's data field bytes are given (packed, split-packed or unpacked)."""
    return field_bytes(1, field_scalar(1, rows) + field_scalar(2, columns) + data_field) + field_scalar(2, shard_index)


def parse_matrix(b, begin, end):
    """(row_count, col_count, data): uint32 fields keep their low 32 bits; data packed or not."""
    rows = columns = 0
    data = []
    for number, wire, value in fields(b, begin, end):
        if number == 1:
            rows = value & 0xffffffff
        elif number == 2:
            columns = value & 0xffffffff
        elif number == 3:
            if wire == 0:
                data.append(value)
            elif wire == LEN:
                p, to = value
                while p < to:
                    v, p = read_varint(b, p, to)
                    data.append(v)
            else:
                raise ProtoError("invalid", "malformedProtobuf: data wire type")
    return rows, columns, data


def parse_request(b):
    """-> (matrix or None, shard_index, configuration_hash)"""
    matrix, shard, digest = None, 0, b""
    for number, wire, value in fields(b, 0, len(b)):
        if number == 1:
            if matrix is not None:
                raise ProtoError("invalid", "malformedProtobuf: a singular message given twice")
            matrix = parse_matrix(b, *value)
        elif number == 2:
            shard = value & 0xffffffff
        elif number == 3:
            digest = b[value[0]:value[1]]
    return matrix, shard, digest


def parse_response(b):
    for number, wire, value in fields(b, 0, len(b)):
        if number == 1:
            return parse_matrix(b, *value)
    return None


def encode_encryption_params(n, error_std_dev, pt, ct):
    return (field_scalar(1, n) + (varint(2 << 3 | FIXED64) + struct.pack("<d", error_std_dev) if error_std_dev else b"") +
            field_scalar(3, pt) + field_scalar(4, ct))


def encode_params(n, error_std_dev, pt, ct, seed, entry_size, entries_per_column, chunks_per_entry, columns):
    """SimplePirParameters.proto()"""
    return (field_bytes(1, encode_encryption_params(n, error_std_dev, pt, ct)) + (field_bytes(2, seed) if seed else b"") +
            field_scalar(3, entry_size) + field_scalar(4, entries_per_column) + field_scalar(5, chunks_per_entry) +
            field_scalar(6, columns))


def encode_database_mapping(entries, chunk_size):
    """entries: (original_index, size, [(shard_index, index)])"""
    out = b""
    for index, size, chunks in entries:
        body = field_scalar(1, index) + field_scalar(2, size)
        body += b"".join(field_bytes(3, field_scalar(1, s) + field_scalar(2, i)) for s, i in chunks)
        out += field_bytes(1, body)
    return out + field_scalar(2, chunk_size)


def encode_config(entries, chunk_size, params, hint_identifiers):
    """params: encode_params argument tuples"""
    return (field_bytes(1, encode_database_mapping(entries, chunk_size)) +
            b"".join(field_bytes(2, encode_params(*p)) for p in params) +
            b"".join(field_bytes(3, h) for h in hint_identifiers))


def response_capacity(rows, columns, ct):
    """The library's slot for a response of rows x columns values below 2^ct: every varint ceil(ct / 7) bytes."""
    data = rows * columns * -(-ct // 7)
    body = (1 + len(varint(rows)) if rows else 0) + 1 + len(varint(columns)) + (1 + len(varint(data)) + data if rows else 0)
    return 1 + len(varint(body)) + body


def b_offset(q, c, col_tiles):
    tile = (q // 8) * col_tiles + c // 32
    cc = c % 32
    lane = (q % 8) * 4 + (cc % 16) // 4
    return tile * 256 + lane * 8 + (cc // 16) * 4 + cc % 4
