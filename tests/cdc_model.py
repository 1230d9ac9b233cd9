"""--cdcstats on the host: content-defined chunks of each block and their dedupe counts.

The gear table is gear[i] = mix(GEAR_TAG + i). The hash of position p of a block is
h(p) = sum over k = 0..63 of gear[b[p - k]] << k (mod 2^64), bytes before the block counting as
absent. With AVG = 2^bits, MIN = AVG / 4 and MAX = 4 * AVG, strict(p) holds when the top bits + 2
bits of h(p) are zero and loose(p) when the top bits - 2 are. A chunk from c is the least l in
[MIN, AVG) with strict(c + l - 1), else the least l in [AVG, MAX) with loose(c + l - 1), else MAX,
and at most what is left of the block. Every block is chunked on its own from its first byte. Two
chunks are the same when their keys are: the first 16 bytes of their BLAKE3-256 digests with bit 0
set (the key of --dedupestats).
"""
import blake3
import numpy as np

from tests.verify_random_model import mix

GEAR_TAG = 0x6A09E667F3BCC908
M64 = (1 << 64) - 1
GEAR = np.array([mix((GEAR_TAG + i) & M64) for i in range(256)], dtype=np.uint64)


def hashes(block):
    """h(p) of every position of block (uint64), in six doubling passes:
    H_2m(p) = H_m(p) + (H_m(p - m) << m)"""
    h = GEAR[np.frombuffer(bytes(block), dtype=np.uint8)]
    m = 1
    while m < 64:
        shifted = np.zeros_like(h)
        shifted[m:] = h[:-m] << np.uint64(m)
        h = h + shifted
        m *= 2
    return h


def hash_at(block, p):
    """h(p) straight from the definition"""
    return sum(int(GEAR[block[p - k]]) << k for k in range(64) if p - k >= 0) & M64


def cut_lengths(block, avg):
    """the lengths of the chunks of one block at mean chunk size avg"""
    n = len(block)
    bits = avg.bit_length() - 1
    lo_len, hi_len = avg // 4, avg * 4
    h = hashes(block)
    strict = np.flatnonzero(h < np.uint64(1 << (62 - bits)))
    loose = np.flatnonzero(h < np.uint64(1 << (66 - bits)))
    lengths = []
    c = 0
    while c < n:
        last = min(c + hi_len, n) - 1
        lo, mid = c + lo_len - 1, c + avg - 1
        cut = last
        if lo < last:
            i = np.searchsorted(strict, lo)
            if i < len(strict) and strict[i] < min(mid, last):
                cut = int(strict[i])
            else:
                j = np.searchsorted(loose, mid)
                if j < len(loose) and loose[j] < last:
                    cut = int(loose[j])
        lengths.append(cut + 1 - c)
        c = cut + 1
    return lengths


def chunks(data, block_size, avg):
    """the chunks of data read in blocks of block_size, as (offset, length)"""
    out = []
    for start in range(0, len(data), block_size):
        block = data[start:start + block_size]
        offset = start
        for length in cut_lengths(block, avg):
            out.append((offset, length))
            offset += length
    return out


def key(piece):
    """the table key of a chunk"""
    k = bytearray(blake3.blake3(bytes(piece)).digest()[:16])
    k[0] |= 1
    return bytes(k)


def counts(datas, block_size, avg):
    """(N, D, B, U) of the chunks of each of datas read in blocks of block_size: chunks, distinct
    chunks, their bytes, and the bytes of the distinct chunks each counted once"""
    n = b = 0
    distinct = {}
    for data in datas:
        data = bytes(data)
        for offset, length in chunks(data, block_size, avg):
            n += 1
            b += length
            distinct.setdefault(key(data[offset:offset + length]), length)
    return n, len(distinct), b, sum(distinct.values())


def ratio(num, den):
    """the ratio of the console line: two decimals, 1.00 when den is 0"""
    return "%.2f" % (num / den if den else 1.0)


def line(avg, n, d, b, u):
    """the console line of --cdcstats"""
    return ("CDC: %d chunks of %d to %d bytes, mean %d, %d distinct: %d bytes, %d distinct bytes: "
            "%s:1" % (n, avg // 4, avg * 4, b // n if n else 0, d, b, u, ratio(b, u)))
