"""--cdcreducestats on the host: the data reduction of storing each distinct content-defined chunk
once, compressed.

The chunks are those of --cdcstats (tests/cdc_model.py), two chunks are the same when their keys
(the key of --dedupestats and --reducestats) are, and each distinct chunk is stored as
min(LZ4 size, length) by the parse of --compressstats (tests/compress_model.py).
"""
from tests import cdc_model, compress_model
from tests.reduce_model import ratio


def distinct(datas, block_size, avg):
    """(N, B, {key: (length, stored)}) of the chunks of each of datas read in blocks of
    block_size"""
    n = b = 0
    out = {}
    for data in datas:
        data = bytes(data)
        for offset, length in cdc_model.chunks(data, block_size, avg):
            n += 1
            b += length
            piece = data[offset:offset + length]
            key = cdc_model.key(piece)
            if key not in out:
                out[key] = (length, min(compress_model.size(piece), length))
    return n, b, out


def counts(datas, block_size, avg):
    """(N, D, B, U, S) of the chunks of each of datas read in blocks of block_size: chunks,
    distinct chunks, their bytes, the bytes of the distinct chunks each counted once, and those
    stored compressed"""
    n, b, table = distinct(datas, block_size, avg)
    u = sum(length for length, _ in table.values())
    s = sum(stored for _, stored in table.values())
    return n, len(table), b, u, s


def line(avg, n, d, b, u, s):
    """the console line of --cdcreducestats"""
    return ("CDC reduce: %d chunks of %d to %d bytes, mean %d, %d distinct: %d bytes, %d distinct "
            "bytes stored as %d: dedupe %s:1, compress %s:1, total %s:1" %
            (n, avg // 4, avg * 4, b // n if n else 0, d, b, u, s, ratio(b, u), ratio(u, s),
             ratio(b, s)))
