"""CPU restatement of --verifyrandgrain: the content of a file position is byte (position mod G)
of the random fill (the CPU oracle's orc_fill_random_ctr) of a block of length G whose block
counter is the position counter of the grain's offset. Positions wrap at 2^64."""
import functools

import numpy as np

from tests import kernel_cases as kc
from tests import oracle_lib
from tests import verify_random_model as vrm

U64 = vrm.U64


ORACLE_MAX_GRAIN = 1 << 20


@functools.lru_cache(maxsize=256)
def grain_bytes(grain, pct, seed, file_key, grain_offset):
    """the whole grain at file position grain_offset (a multiple of grain)"""
    return oracle_lib.fill_random_ctr(grain, pct, seed, vrm.pos_counter(file_key, grain_offset))


def content(start, length, grain, pct, seed, file_key):
    """bytes of file positions [start, start + length), mod 2^64. Grains of up to 1 MiB come
    whole from the oracle; of larger ones only the slice is built, by the numpy closed form of
    the same fill (tests/kernel_cases.py, itself checked against the oracle)."""
    out = bytearray()
    pos, end = start, start + length
    while pos < end:
        p = pos & U64
        q = p & (grain - 1)
        n = min(grain - q, end - pos)
        if grain <= ORACLE_MAX_GRAIN:
            out += grain_bytes(grain, pct, seed, file_key, p - q)[q:q + n]
        else:
            out += kc.random_bytes(grain, pct, seed, vrm.pos_counter(file_key, p - q), q,
                                   n).tobytes()
        pos += n
    return bytes(out)


def file_content(size, grain, pct, seed, file_key):
    return content(0, size, grain, pct, seed, file_key)


def error_text(data, grain, pct, seed, file_key):
    """the worker's verification error for the first bad byte of file content data, or None"""
    want = np.frombuffer(file_content(len(data), grain, pct, seed, file_key), dtype=np.uint8)
    bad = np.flatnonzero(np.frombuffer(bytes(data), dtype=np.uint8) != want)
    if not len(bad):
        return None
    i = int(bad[0])
    return ("Data verification failed. Offset: %d; Expected value: %d; Actual value: %d"
            % (i, want[i], data[i]))
