"""An independent model of the reflected CRCs behind --checksumalgo, for the tests, generic over the
width and the polynomial.

R(M) is the raw reflected CRC (register 0 at the start, no final XOR), computed bit by bit. X(c, n)
appends n zero bytes to c's message: c * x^(8n) mod P, by carry-less multiplication of the
polynomials in ordinary bit order and reduction by the full polynomial of width + 1 bits, with x^n
by plain square-and-multiply over all bits of n (no reduction of n by the order of x). The
published CRC is R ^ X(all ones, |M|) ^ all ones. The tests check it against zlib.crc32 and the
published vectors of each algorithm."""
import dataclasses


@dataclasses.dataclass(frozen=True)
class Algo:
    name: str
    width: int
    poly_reflected: int

    @property
    def mask(self):
        return (1 << self.width) - 1

    @property
    def poly_normal(self):
        """x^width + ... + 1, bit k = coefficient of x^k"""
        return (1 << self.width) | int(f"{self.poly_reflected:0{self.width}b}"[::-1], 2)

    @property
    def digits(self):
        return self.width // 4


ALGOS = {
    "crc32": Algo("crc32", 32, 0xEDB88320),
    "crc32c": Algo("crc32c", 32, 0x82F63B78),
    "crc64nvme": Algo("crc64nvme", 64, 0x9A6C9329AC4BC9B5),
}


def raw_crc(algo, data, crc=0):
    """R(previous message || data), crc = R(previous message)"""
    for byte in data:
        crc ^= byte
        for _ in range(8):
            crc = (crc >> 1) ^ (algo.poly_reflected if crc & 1 else 0)
    return crc


def _reflect(algo, value):
    return int(f"{value:0{algo.width}b}"[::-1], 2)


def _polymulmod(algo, a, b):
    """a * b mod P in ordinary bit order"""
    prod = 0
    while b:
        if b & 1:
            prod ^= a
        b >>= 1
        a <<= 1
    for bit in range(prod.bit_length() - 1, algo.width - 1, -1):
        if prod >> bit & 1:
            prod ^= algo.poly_normal << (bit - algo.width)
    return prod


def _xpow(algo, n):
    """x^n mod P in ordinary bit order"""
    result, base = 1, 2
    while n:
        if n & 1:
            result = _polymulmod(algo, result, base)
        base = _polymulmod(algo, base, base)
        n >>= 1
    return result


def shift(algo, crc, num_zero_bytes):
    """X(crc, n) = R(crc's message || n zero bytes)"""
    return _reflect(algo, _polymulmod(algo, _reflect(algo, crc), _xpow(algo, 8 * num_zero_bytes)))


def finish(algo, raw, size):
    """the published CRC of a message of size bytes from its R"""
    return raw ^ shift(algo, algo.mask, size) ^ algo.mask


def crc(algo, data):
    return finish(algo, raw_crc(algo, data), len(data))


def contribution(algo, block, offset, file_size):
    """what a block at offset of a file of file_size adds (XOR) to the file's R"""
    return shift(algo, raw_crc(algo, block), file_size - offset - len(block))


def file_raw_crc(algo, data, parts):
    """R of data from the contributions of parts [(offset, length)] that cover it once"""
    raw = 0
    for offset, length in parts:
        raw ^= contribution(algo, data[offset:offset + length], offset, len(data))
    return raw


def order_of_x(algo):
    """the order of x mod P that the library reduces shifts by (checked by the tests)"""
    return {"crc32": (1 << 32) - 1, "crc32c": (1 << 31) - 1, "crc64nvme": (1 << 64) - 1}[algo.name]
