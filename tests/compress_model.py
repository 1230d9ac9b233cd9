"""Model of the --compressstats LZ4 parse (DESIGN.md "--compressstats") and an LZ4 block decoder
written from the LZ4 block format.

The candidate of a position (the latest earlier position of the same 12-bit hash) does not depend
on the parse, so every position that can take a match is found with numpy first, and the greedy
walk jumps from one such position to the next."""
import numpy as np

HASH_MUL = 2654435761
MAX_OFFSET = 65535


def _ext(x):
    return 0 if x < 15 else (x - 15) // 255 + 1


def _match_positions(b):
    """the positions p <= n - 12 whose candidate is at most MAX_OFFSET back and has the same 4
    bytes, and their candidates"""
    n = len(b)
    last = n - 12
    a = np.frombuffer(b, dtype=np.uint8).astype(np.uint32)
    vals = a[:last + 1] | (a[1:last + 2] << 8) | (a[2:last + 3] << 16) | (a[3:last + 4] << 24)
    hashes = ((vals.astype(np.uint64) * HASH_MUL) & 0xffffffff) >> 20
    order = np.argsort(hashes, kind="stable")  # (stable: positions ascend within a hash)
    same = hashes[order[1:]] == hashes[order[:-1]]
    cand = np.full(last + 1, -1, dtype=np.int64)
    cand[order[1:][same]] = order[:-1][same]
    pos = np.arange(last + 1, dtype=np.int64)
    ok = (cand >= 0) & (pos - cand <= MAX_OFFSET)
    ok[ok] = vals[cand[ok]] == vals[pos[ok]]
    return pos[ok], cand[ok]


def _extend(b, p, q, end):
    """the match length at p against q, ending before byte end"""
    length, step = 4, 16
    while p + length < end:
        step = min(step, end - p - length)
        if b[q + length:q + length + step] == b[p + length:p + length + step]:
            length += step
            step *= 2
            continue
        while b[q + length] == b[p + length]:  # (a mismatch lies within step)
            length += 1
        return length
    return length


def parse(b):
    """the sequences of chunk b: [(literal start, literal count, offset, match length)], the last
    one without a match (offset and match length 0)"""
    b = bytes(b)
    n = len(b)
    seqs = []
    anchor = 0
    if n >= 13:
        positions, cands = _match_positions(b)
        i = 0
        while i < len(positions):
            p, q = int(positions[i]), int(cands[i])
            length = _extend(b, p, q, n - 5)
            seqs.append((anchor, p - anchor, p - q, length))
            anchor = p + length
            i = int(np.searchsorted(positions, anchor))
    seqs.append((anchor, n - anchor, 0, 0))
    return seqs


def size(b):
    """the LZ4 block size of chunk b"""
    total = 0
    for _, lits, offset, length in parse(b):
        total += 1 + _ext(lits) + lits + (2 + _ext(length - 4) if length else 0)
    return total


def _ext_bytes(x):
    if x < 15:
        return b""
    r = x - 15
    return b"\xff" * (r // 255) + bytes([r % 255])


def compress(b):
    """the LZ4 block of chunk b"""
    b = bytes(b)
    out = bytearray()
    for start, lits, offset, length in parse(b):
        out.append((min(lits, 15) << 4) | (min(length - 4, 15) if length else 0))
        out += _ext_bytes(lits)
        out += b[start:start + lits]
        if length:
            out += offset.to_bytes(2, "little")
            out += _ext_bytes(length - 4)
    return bytes(out)


def check_block_rules(b):
    """the rules that make any LZ4 decoder accept the block: offsets 1..65535, the last 5 bytes
    literals, no match starting past n - 12"""
    n = len(b)
    for start, lits, offset, length in parse(b):
        if not length:
            continue
        p = start + lits
        assert 1 <= offset <= MAX_OFFSET
        assert p <= n - 12
        assert p + length <= n - 5


def decode(block, max_out=1 << 31):
    """an LZ4 block decoder (LZ4 block format): token, literal length bytes, literals, 2-byte
    offset, match length bytes; the last sequence has literals only"""
    block = bytes(block)
    out = bytearray()
    i = 0

    def length(nibble):
        nonlocal i
        x = nibble
        if nibble == 15:
            while True:
                c = block[i]
                i += 1
                x += c
                if c != 255:
                    break
        return x

    while True:
        token = block[i]
        i += 1
        lits = length(token >> 4)
        if i + lits > len(block):
            raise ValueError("literals past the end of the block")
        out += block[i:i + lits]
        i += lits
        if i == len(block):
            break
        offset = block[i] | (block[i + 1] << 8)
        i += 2
        if not 0 < offset <= len(out):
            raise ValueError("offset %d out of range" % offset)
        ml = length(token & 15) + 4
        start = len(out) - offset
        if offset >= ml:
            out += out[start:start + ml]
        else:
            pattern = bytes(out[start:])
            out += (pattern * (ml // offset + 1))[:ml]
        if len(out) > max_out:
            raise ValueError("output too long")
    return bytes(out)


def chunk_sizes(data, chunk):
    """[(chunk length, LZ4 size)] of the chunks of data"""
    return [(len(data[o:o + chunk]), size(data[o:o + chunk])) for o in range(0, len(data), chunk)]


def counts(datas, chunk):
    """(chunks, bytes, bytes stored, incompressible) of the chunks of each of datas"""
    n = b_in = stored = incompressible = 0
    for data in datas:
        for length, s in chunk_sizes(data, chunk):
            n += 1
            b_in += length
            stored += min(s, length)
            incompressible += s >= length
    return n, b_in, stored, incompressible
