"""An independent model of the CRC-32 arithmetic behind --checksums, for the tests.

R(M) is the raw reflected CRC-32 (polynomial 0xEDB88320, register 0 at the start, no final XOR),
computed bit by bit. X(c, n) appends n zero bytes to c's message: c * x^(8n) mod P, by carry-less
multiplication of the polynomials in ordinary bit order and reduction by the full 33-bit
polynomial. zlib's CRC-32 follows from R and X; the tests check all three against zlib.crc32."""
import random

POLY_REFLECTED = 0xEDB88320
POLY_NORMAL = 0x104C11DB7  # x^32 + ... + 1, bit k = coefficient of x^k


def raw_crc(data, crc=0):
    """R(previous message || data), crc = R(previous message)"""
    for byte in data:
        crc ^= byte
        for _ in range(8):
            crc = (crc >> 1) ^ (POLY_REFLECTED if crc & 1 else 0)
    return crc


def _reflect32(value):
    return int(f"{value:032b}"[::-1], 2)


def _polymulmod(a, b):
    """a * b mod P in ordinary bit order"""
    prod = 0
    while b:
        if b & 1:
            prod ^= a
        b >>= 1
        a <<= 1
    for bit in range(prod.bit_length() - 1, 31, -1):
        if prod >> bit & 1:
            prod ^= POLY_NORMAL << (bit - 32)
    return prod


def _xpow(n):
    """x^n mod P in ordinary bit order"""
    result, base = 1, 2
    while n:
        if n & 1:
            result = _polymulmod(result, base)
        base = _polymulmod(base, base)
        n >>= 1
    return result


def shift(crc, num_zero_bytes):
    """X(crc, n) = R(crc's message || n zero bytes)"""
    return _reflect32(_polymulmod(_reflect32(crc), _xpow(8 * num_zero_bytes)))


def finish(raw, size):
    """zlib's CRC-32 of a message of size bytes from its R"""
    return raw ^ shift(0xFFFFFFFF, size) ^ 0xFFFFFFFF


def contribution(block, offset, file_size):
    """what a block at offset of a file of file_size adds (XOR) to the file's R"""
    return shift(raw_crc(block), file_size - offset - len(block))


def random_split(size, rng):
    """[(offset, length)] that cover [0, size) exactly once, in random order: up to a dozen random
    cuts, one block of 1 byte (size > 0) and two blocks of 0 bytes"""
    cuts = set(rng.sample(range(size + 1), min(size + 1, rng.randint(0, 12))))
    if size:
        one = rng.randrange(size)
        cuts |= {one, one + 1}
    bounds = sorted(cuts | {0, size})
    parts = [(lo, hi - lo) for lo, hi in zip(bounds, bounds[1:])]
    parts += [(rng.randint(0, size), 0) for _ in range(2)]
    rng.shuffle(parts)
    return parts


def file_raw_crc(data, parts):
    crc = 0
    for offset, length in parts:
        crc ^= contribution(data[offset:offset + length], offset, len(data))
    return crc

