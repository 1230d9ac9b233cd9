"""Writes blake3_vectors.json: BLAKE3-256 digests, from the `blake3` package, of the i mod 251
byte pattern at the lengths of BLAKE3's published test vectors and at a few MiB-scale sizes with
odd tails. Tests use these digests where the package may be missing (on the GPU machine)."""

import json
import os

import blake3
import numpy as np

LENGTHS = [0, 1, 1023, 1024, 1025, 2048, 2049, 3072, 3073, 4096, 4097, 5120, 5121, 6144, 6145,
           7168, 7169, 8192, 8193, 16384, 31744, 102400,
           63, 64, 65, 127, 128, 129,
           (1 << 20) + 1, 3 * (1 << 20) - 1023, (5 << 20) + 777, (8 << 20) + 1024 * 3 + 5]


def pattern(n):
    return (np.arange(n, dtype=np.uint64) % 251).astype(np.uint8).tobytes()


def main():
    vectors = [{"length": n, "digest": blake3.blake3(pattern(n)).hexdigest()}
               for n in sorted(set(LENGTHS))]
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "blake3_vectors.json")
    with open(path, "w") as f:
        json.dump({"pattern": "i mod 251", "vectors": vectors}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
