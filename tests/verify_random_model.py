"""CPU restatement of --verifyrand (plain Python + numpy, no product headers): the position
counter and the two fileKey forms of elb_patterns.cuh, and a reference verify of a random-filled
block whose expected bytes come from the CPU oracle's counter-based fill (orc_fill_random_ctr)."""
import numpy as np

from tests import oracle_lib

U64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15


def mix(z):
    """SplitMix64 finaliser on a Python int"""
    z &= U64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & U64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & U64
    return z ^ (z >> 31)


def pos_counter(file_key, file_offset):
    """block counter of the block at file_offset of the file with file_key"""
    return mix(mix(file_key + GOLDEN) ^ (file_offset & U64))


def dir_file_key(rank, dir_index, file_index):
    """file_key of the dir mode file r<rank>/d<dir_index>/r<rank>-f<file_index>"""
    return mix(mix(mix(rank) + dir_index) + file_index)


def random_block(length, pct, seed, counter):
    return np.frombuffer(oracle_lib.fill_random_ctr(length, pct, seed, counter), dtype=np.uint8)


def verify_random(data, pct, seed, counter):
    """(numMismatchBytes, firstMismatchIdx) of data against the random fill of its length"""
    got = np.frombuffer(bytes(data), dtype=np.uint8)
    bad = np.flatnonzero(got != random_block(len(got), pct, seed, counter))
    return (len(bad), int(bad[0]) if len(bad) else U64)


def file_random_content(size, block, pct, seed, file_key):
    """expected bytes of a whole file written with --verifyrand seed, -b block, -s size"""
    out = bytearray()
    for off in range(0, size, block):
        n = min(block, size - off)
        out += random_block(n, pct, seed, pos_counter(file_key, off)).tobytes()
    return bytes(out)


def error_text(data, block, pct, seed, file_key):
    """the worker's verification error for the first bad byte of file content data (blocks in file
    order), or None if the data is clean"""
    for off in range(0, len(data), block):
        chunk = data[off:off + block]
        want = random_block(len(chunk), pct, seed, pos_counter(file_key, off))
        bad = np.flatnonzero(np.frombuffer(chunk, dtype=np.uint8) != want)
        if len(bad):
            i = int(bad[0])
            return ("Data verification failed. Offset: %d; Expected value: %d; Actual value: %d"
                    % (off + i, want[i], chunk[i]))
    return None
