"""An independent BLAKE3 model (default hash, 256-bit output), written from the BLAKE3
specification and vectorised with numpy across chunks and parents, so that it hashes tens of MiB
in a test's time. The kernel's and the library's results are checked against it."""

import numpy as np

IV = np.array([0x6A09E667, 0xBB67AE85, 0x3C6EF372, 0xA54FF53A,
               0x510E527F, 0x9B05688C, 0x1F83D9AB, 0x5BE0CD19], dtype=np.uint32)
PERMUTATION = [2, 6, 3, 10, 7, 0, 4, 13, 1, 11, 12, 5, 9, 14, 15, 8]
CHUNK_START, CHUNK_END, PARENT, ROOT = 1, 2, 4, 8
CHUNK_BYTES = 1024


def _rotr(x, n):
    return (x >> np.uint32(n)) | (x << np.uint32(32 - n))


def _g(v, a, b, c, d, mx, my):
    v[a] = v[a] + v[b] + mx
    v[d] = _rotr(v[d] ^ v[a], 16)
    v[c] = v[c] + v[d]
    v[b] = _rotr(v[b] ^ v[c], 12)
    v[a] = v[a] + v[b] + my
    v[d] = _rotr(v[d] ^ v[a], 8)
    v[c] = v[c] + v[d]
    v[b] = _rotr(v[b] ^ v[c], 7)


def compress(cv, m, counter, block_len, flags):
    """the first 8 output words of the compression of N blocks at once: cv (N, 8), m (N, 16)
    uint32, counter (N,) uint64, block_len and flags (N,) or scalars"""
    n = cv.shape[0]
    counter = np.broadcast_to(np.asarray(counter, dtype=np.uint64), (n,))
    v = [cv[:, i].copy() for i in range(8)] + [np.full(n, IV[i], dtype=np.uint32) for i in range(4)]
    v += [(counter & np.uint64(0xFFFFFFFF)).astype(np.uint32), (counter >> np.uint64(32)).astype(np.uint32),
          np.broadcast_to(np.asarray(block_len, dtype=np.uint32), (n,)).copy(),
          np.broadcast_to(np.asarray(flags, dtype=np.uint32), (n,)).copy()]
    words = [m[:, i] for i in range(16)]
    with np.errstate(over="ignore"):
        for rnd in range(7):
            _g(v, 0, 4, 8, 12, words[0], words[1])
            _g(v, 1, 5, 9, 13, words[2], words[3])
            _g(v, 2, 6, 10, 14, words[4], words[5])
            _g(v, 3, 7, 11, 15, words[6], words[7])
            _g(v, 0, 5, 10, 15, words[8], words[9])
            _g(v, 1, 6, 11, 12, words[10], words[11])
            _g(v, 2, 7, 8, 13, words[12], words[13])
            _g(v, 3, 4, 9, 14, words[14], words[15])
            if rnd < 6:
                words = [words[PERMUTATION[i]] for i in range(16)]
    return np.stack([v[i] ^ v[i + 8] for i in range(8)], axis=1)


def _cv_bytes(cv):
    return np.ascontiguousarray(cv, dtype="<u4").tobytes()


def chunk_cvs(data, first_counter=0, root=False):
    """(N, 8) CVs of the 1 KiB chunks of data (the last may be short; no data: one empty chunk),
    chunk i with counter first_counter + i. root: data is one chunk, its CV is the digest."""
    data = np.frombuffer(bytes(data), dtype=np.uint8)
    num_chunks = max(1, -(-len(data) // CHUNK_BYTES))
    tail_len = len(data) - (num_chunks - 1) * CHUNK_BYTES
    padded = np.zeros(num_chunks * CHUNK_BYTES, dtype=np.uint8)
    padded[:len(data)] = data
    words = padded.view("<u4").reshape(num_chunks, 16, 16)
    counters = np.uint64(first_counter) + np.arange(num_chunks, dtype=np.uint64)
    cvs = np.tile(IV, (num_chunks, 1))
    num_full = num_chunks if tail_len == CHUNK_BYTES else num_chunks - 1

    if num_full:
        for b in range(16):
            flags = (CHUNK_START if b == 0 else 0) | (CHUNK_END if b == 15 else 0)
            if b == 15 and root:
                flags |= ROOT
            cvs[:num_full] = compress(cvs[:num_full], words[:num_full, b], counters[:num_full],
                                      64, flags)

    if num_full < num_chunks:  # the short last chunk
        blocks = max(1, -(-tail_len // 64))
        cv = cvs[-1:].copy()
        for b in range(blocks):
            flags = (CHUNK_START if b == 0 else 0) | (CHUNK_END if b == blocks - 1 else 0)
            if b == blocks - 1 and root:
                flags |= ROOT
            cv = compress(cv, words[-1:, b], counters[-1:], min(64, tail_len - 64 * b), flags)
        cvs[-1:] = cv

    return cvs


def parents(left, right, root=False):
    """(N, 8) parents of the (N, 8) CVs left and right"""
    m = np.concatenate([left, right], axis=1)
    return compress(np.tile(IV, (left.shape[0], 1)), m, 0, 64, PARENT | (ROOT if root else 0))


def parent(left, right, root=False):
    """the parent of two 32-byte CVs, as 32 bytes"""
    l = np.frombuffer(bytes(left), dtype="<u4").reshape(1, 8)
    r = np.frombuffer(bytes(right), dtype="<u4").reshape(1, 8)
    return _cv_bytes(parents(l, r, root))


def _subtree(cvs, root):
    """the CV (root: digest) of the tree over the chunk CVs cvs (N, 8), N >= 1"""
    if len(cvs) == 1:
        return cvs[0:1]
    if len(cvs) & (len(cvs) - 1) == 0:
        while len(cvs) > 2:
            cvs = parents(cvs[0::2], cvs[1::2])
        return parents(cvs[0:1], cvs[1:2], root)
    left = 1 << ((len(cvs) - 1).bit_length() - 1)
    return parents(_subtree(cvs[:left], False), _subtree(cvs[left:], False), root)


def run_cv(data, first_chunk):
    """the 32-byte CV of the aligned run of chunks that data (2^j chunks, the last maybe short)
    holds, starting at chunk index first_chunk of its message; not the whole message"""
    return _cv_bytes(_subtree(chunk_cvs(data, first_chunk), False))


def digest(data):
    """BLAKE3-256 of data, 32 bytes"""
    data = bytes(data)
    if len(data) <= CHUNK_BYTES:
        return _cv_bytes(chunk_cvs(data, 0, root=True))
    return _cv_bytes(_subtree(chunk_cvs(data), True))


def chunk_digests(data, chunk_size):
    """[BLAKE3-256 of each chunk_size (a power of two, 2 KiB or more) piece of data], each piece a
    message of its own; the full pieces are hashed together"""
    data = bytes(data)
    num_full = len(data) // chunk_size
    per = chunk_size // CHUNK_BYTES
    out = []
    if num_full:
        counters = np.tile(np.arange(per, dtype=np.uint64), num_full)  # (each piece's own)
        words = np.frombuffer(data[:num_full * chunk_size], dtype="<u4").reshape(-1, 16, 16)
        cvs = np.tile(IV, (len(words), 1))
        for b in range(16):
            flags = (CHUNK_START if b == 0 else 0) | (CHUNK_END if b == 15 else 0)
            cvs = compress(cvs, words[:, b], counters, 64, flags)
        cvs = cvs.reshape(num_full, per, 8)
        while cvs.shape[1] > 2:
            flat_l = cvs[:, 0::2].reshape(-1, 8)
            flat_r = cvs[:, 1::2].reshape(-1, 8)
            cvs = parents(flat_l, flat_r).reshape(num_full, -1, 8)
        roots = parents(cvs[:, 0], cvs[:, 1], root=True)
        out = [_cv_bytes(roots[i:i + 1]) for i in range(num_full)]
    if len(data) > num_full * chunk_size:
        out.append(digest(data[num_full * chunk_size:]))
    return out


def canonical_runs(begin, end):
    """the maximal aligned runs (first chunk, chunk count) of the chunks [begin, end), in order"""
    runs = []
    pos = begin
    while pos < end:
        size = 1
        while pos % (2 * size) == 0 and pos + 2 * size <= end:
            size *= 2
        runs.append((pos, size))
        pos += size
    return runs


def fold_runs(num_chunks):
    """the runs whose CVs blake3_fold joins for a file of num_chunks >= 2 chunks"""
    if num_chunks & (num_chunks - 1) == 0:
        half = num_chunks // 2
        return [(0, half), (half, half)]
    return canonical_runs(0, num_chunks)


def pattern(n):
    """the i mod 251 bytes of BLAKE3's published test vectors"""
    return (np.arange(n, dtype=np.uint64) % 251).astype(np.uint8).tobytes()
