"""--reducestats on the host: the data reduction of storing each distinct chunk once, compressed.

A chunk is a K-piece of a file, the last one possibly short. Two chunks are the same when their
keys are: the first 16 bytes of the chunk's BLAKE3-256 digest with bit 0 set (the key of
--dedupestats). Each distinct chunk is stored as min(LZ4 size, length) by the parse of
--compressstats.
"""
from tests import blake3_model, compress_model


def chunk_keys(data, chunk):
    """the key of each chunk of data"""
    keys = []
    for digest in blake3_model.chunk_digests(data, chunk):
        key = bytearray(digest[:16])
        key[0] |= 1
        keys.append(bytes(key))
    return keys


def counts(datas, chunk):
    """(N, D, B, U, S) of the K-chunks of each of datas: chunks, distinct chunks, their bytes, the
    bytes of the distinct chunks each counted once, and those stored compressed"""
    n = b = 0
    distinct = {}
    for data in datas:
        data = bytes(data)
        for j, key in enumerate(chunk_keys(data, chunk)):
            piece = data[j * chunk:(j + 1) * chunk]
            n += 1
            b += len(piece)
            if key not in distinct:
                distinct[key] = (len(piece), min(compress_model.size(piece), len(piece)))
    u = sum(length for length, _ in distinct.values())
    s = sum(stored for _, stored in distinct.values())
    return n, len(distinct), b, u, s


def ratio(num, den):
    """a ratio of the console line: two decimals, 1.00 when den is 0"""
    return "%.2f" % (num / den if den else 1.0)


def line(chunk, n, d, b, u, s):
    """the console line of --reducestats"""
    return ("Reduce: %d chunks of %d, %d distinct: %d bytes, %d distinct bytes stored as %d: "
            "dedupe %s:1, compress %s:1, total %s:1" %
            (n, chunk, d, b, u, s, ratio(b, u), ratio(u, s), ratio(b, s)))
