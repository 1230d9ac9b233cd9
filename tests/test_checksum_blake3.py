"""CPU tests of the BLAKE3 digests: the numpy model (tests/blake3_model.py) against the published
known answers, the goldens and the `blake3` package; the library's parent and fold against the
model and the goldens for random files cut into random blocks of 1 KiB multiples, their runs
joined as a host merge joins them; the argument checks of elb_blake3_chunks; blake3 lists, the
command line's acceptances, rejections and help text, and the config's rejections."""
import ctypes
import json
import os
import random

import pytest

from elbencho_b200 import WorkerConfig, WorkerError, WorkerManager, _native, kernels
from tests import blake3_model as model
from tests.test_cli import run_cli

KiB, MiB = 1 << 10, 1 << 20

EMPTY = "af1349b9f5f9a1a6a0404dea36dcc9499bcb25c9adc112b7cc9a93cae41f3262"
ABC = "6437b3ac38465133ffb63b75273a8db548c558465d79db03fd359c6cd5bd9d85"

with open(os.path.join(os.path.dirname(__file__), "golden", "blake3_vectors.json")) as _f:
    GOLDEN = {v["length"]: v["digest"] for v in json.load(_f)["vectors"]}


def test_model_known_answers():
    assert model.digest(b"").hex() == EMPTY
    assert model.digest(b"abc").hex() == ABC


@pytest.mark.parametrize("length", sorted(GOLDEN))
def test_model_matches_goldens(length):
    assert model.digest(model.pattern(length)).hex() == GOLDEN[length]


def test_model_matches_package():
    blake3 = pytest.importorskip("blake3")
    rng = random.Random(3)
    for size in [rng.randrange(0, 70000) for _ in range(40)] + [rng.randrange(1, 3 * MiB)]:
        data = rng.randbytes(size)
        assert model.digest(data) == blake3.blake3(data).digest(), size
    data = rng.randbytes(MiB + 5000)
    for k in (4 * KiB, 64 * KiB, MiB):
        assert model.chunk_digests(data, k) == [blake3.blake3(data[p:p + k]).digest()
                                               for p in range(0, len(data), k)]


def _merge(runs, num_chunks):
    """join (first, count, cv) runs of a file eagerly, as aligned siblings arrive, never into the
    whole file: what remains are the runs blake3_fold takes"""
    held = {}
    for first, count, cv in runs:
        while True:
            sibling = first + count if first % (2 * count) == 0 else first - count
            if (held.get(sibling, (None,))[0] != count or
                    (min(first, sibling) == 0 and 2 * count == num_chunks)):
                break
            _, other = held.pop(sibling)
            left, right = (cv, other) if sibling > first else (other, cv)
            first, count = min(first, sibling), 2 * count
            cv = kernels.blake3_parent(left, right)
        held[first] = (count, cv)
    return [(first, held[first][0], held[first][1]) for first in sorted(held)]


def _random_blocks(size, rng):
    """random cut points on 1 KiB boundaries, some blocks of non-power-of-two sizes"""
    cuts = sorted({rng.randrange(1, size // KiB) * KiB for _ in range(rng.randrange(1, 12))}
                  if size > 2 * KiB else set())
    bounds = [0] + [c for c in cuts if c < size] + [size]
    return [(bounds[i], bounds[i + 1]) for i in range(len(bounds) - 1)]


@pytest.mark.parametrize("seed", range(12))
def test_fold_of_random_blocks_matches_model(seed):
    rng = random.Random(seed)
    size = rng.choice([rng.randrange(KiB + 1, 70 * KiB), rng.randrange(1, 3 * MiB)])
    size = max(size, KiB + 1)
    data = rng.randbytes(size)
    num_chunks = -(-size // KiB)
    blocks = _random_blocks(size, rng)
    rng.shuffle(blocks)  # any order
    runs = []
    for begin, end in blocks:
        for first, count in model.canonical_runs(begin // KiB, -(-end // KiB)):
            runs.append((first, count, model.run_cv(data[first * KiB:(first + count) * KiB], first)))
    held = _merge(runs, num_chunks)
    assert [(f, c) for f, c, _ in held] == model.fold_runs(num_chunks)
    assert kernels.blake3_fold([cv for _, _, cv in held], size) == model.digest(data)


@pytest.mark.parametrize("length", [n for n in sorted(GOLDEN) if n > KiB])
def test_fold_matches_goldens(length):
    data = model.pattern(length)
    cvs = [model.run_cv(data[f * KiB:(f + c) * KiB], f)
           for f, c in model.fold_runs(-(-length // KiB))]
    assert kernels.blake3_fold(cvs, length).hex() == GOLDEN[length]


def test_parent_matches_model():
    rng = random.Random(5)
    for root in (False, True):
        left, right = rng.randbytes(32), rng.randbytes(32)
        assert kernels.blake3_parent(left, right, root) == model.parent(left, right, root)


def test_fold_rejects_runs_that_do_not_fit():
    cv = bytes(32)
    with pytest.raises(kernels.KernelError, match="3 runs do not make a file of 4096 bytes"):
        kernels.blake3_fold([cv] * 3, 4096)
    with pytest.raises(kernels.KernelError, match="1 runs do not make a file of 1024 bytes"):
        kernels.blake3_fold([cv], 1024)


def test_blake3_chunks_argument_checks():
    lib = _native.load()
    raw = kernels.pack_block_descs([(0x1000, 4096, 0, 0)])
    descs = ctypes.create_string_buffer(raw, len(raw))
    shifts = (ctypes.c_uint64 * 1)(0)
    digests = ctypes.create_string_buffer(32 * 4)
    assert lib.elb_blake3_chunks(descs, None, 1, 11, 1, digests, None, None, None) == -1
    assert _native.last_error() == "elb_blake3_chunks: chunk shift 11 is neither 64 nor in [12, 40]"
    assert lib.elb_blake3_chunks(descs, None, 1, 12, 0, digests, None, None, None) == -1
    assert _native.last_error() == "elb_blake3_chunks: slots per descriptor must be at least 1"
    assert lib.elb_blake3_chunks(descs, None, 1, 64, 1, digests, None, None, None) == -1
    assert _native.last_error() == "elb_blake3_chunks: NULL descriptor, shift or digest array"
    assert lib.elb_blake3_chunks(descs, None, 1, 12, 1, digests, digests, None, None) == -1
    assert _native.last_error() == "elb_blake3_chunks: host digests and device ticket go together"
    # off 1 KiB boundaries: a start, and an end before the file's end
    for offset, length, shift in [(512, 4096, 0), (0, 1536, 100)]:
        raw = kernels.pack_block_descs([(0x1000, length, offset, 0)])
        descs = ctypes.create_string_buffer(raw, len(raw))
        shifts[0] = shift
        assert lib.elb_blake3_chunks(descs, shifts, 1, 64, 4, digests, None, None, None) == -1
        assert _native.last_error() == (
            "elb_blake3_chunks: descriptor 0 (offset %d, length %d) is not on 1 KiB boundaries"
            % (offset, length))
    # chunked: a start off a chunk boundary
    raw = kernels.pack_block_descs([(0x1000, 4096, 1024, 0)])
    descs = ctypes.create_string_buffer(raw, len(raw))
    assert lib.elb_blake3_chunks(descs, None, 1, 12, 4, digests, None, None, None) == -1
    assert "descriptor 0 (offset 1024, length 4096) is not on chunk boundaries" in _native.last_error()
    # more runs than slots: chunks 1 .. 6 are the runs 1, 2-3, 4-5, 6
    raw = kernels.pack_block_descs([(0x1000, 6 * KiB, KiB, 0)])
    descs = ctypes.create_string_buffer(raw, len(raw))
    shifts[0] = 5000
    assert lib.elb_blake3_chunks(descs, shifts, 1, 64, 3, digests, None, None, None) == -1
    assert _native.last_error() == ("elb_blake3_chunks: descriptor 0 (offset 1024, length 6144) "
                                    "needs 4 slots, more than 3 slots per descriptor")
    raw = kernels.pack_block_descs([(0x1000, 8 * KiB, 0, 0)])
    descs = ctypes.create_string_buffer(raw, len(raw))
    assert lib.elb_blake3_chunks(descs, None, 1, 12, 1, digests, None, None, None) == -1
    assert "needs 2 slots, more than 1 slots per descriptor" in _native.last_error()
    assert lib.elb_blake3_chunks(None, None, 0, 12, 1, None, None, None, None) == 0


def test_crc_entries_still_reject_blake3_id():
    lib = _native.load()
    assert lib.elb_crc_finish(3, 0x1234, 5) == 0
    assert _native.last_error() == "elb_crc_finish: unknown checksum algorithm 3"


# ------------------------------------------------------------------------------------------------
# lists, command line and config
# ------------------------------------------------------------------------------------------------

CLI = ["-r", "-b", "256k", "-s", "4m", "--gpuids", "0"]
DIGEST = "0123456789abcdef" * 4


def dry_run(tmp_path, text, *extra):
    lst = tmp_path / "list"
    lst.write_text(text)
    return run_cli("--dryrun", *CLI, *extra, "--checksumverify", str(lst), str(tmp_path / "data"))


@pytest.mark.parametrize("text", [
    "# phase WRITE chunk 65536 blake3\n/a 0 65536 %s\n/a 65536 7 %s\n" % (DIGEST, DIGEST.upper()),
    "# phase WRITE blake3\n/a 4096 4096 %s\n/b 1 1 -\n# phase READ chunk 4096 blake3\n"
    "/a 0 4096 %s\n" % (DIGEST, DIGEST),
])
def test_blake3_lists_parse(tmp_path, text):
    res = dry_run(tmp_path, text)
    assert res.returncode == 0, res.stderr
    res = dry_run(tmp_path, text, "--checksumalgo", "blake3")
    assert res.returncode == 0, res.stderr


@pytest.mark.parametrize("text,line_num", [
    ("# phase WRITE chunk 65536 blake3\n/a 0 65536 %s\n" % DIGEST[:-1], 2),
    ("# phase WRITE chunk 65536 blake3\n\n/a 0 65536 %s0\n" % DIGEST, 3),
    ("# phase WRITE chunk 65536 blake3\n/a 0 65536 0000abcd\n", 2),
    ("# phase WRITE chunk 65536 blake3\n/a 0 65536 %sg\n" % DIGEST[:-1], 2),
])
def test_malformed_blake3_lines_name_their_line(tmp_path, text, line_num):
    res = dry_run(tmp_path, text)
    assert res.returncode == 1
    assert ('Checksum list line %d: not "path offset length blake3": ' % line_num) in res.stderr, \
        res.stderr


@pytest.mark.parametrize("given,listed", [("blake3", "crc32c"), ("crc32", "blake3")])
def test_explicit_algorithm_must_match_a_blake3_list(tmp_path, given, listed):
    digest = DIGEST if listed == "blake3" else "0000abcd"
    text = "# phase WRITE chunk 65536 %s\n/a 0 65536 %s\n" % (listed, digest)
    res = dry_run(tmp_path, text, "--checksumalgo", given)
    assert res.returncode == 1
    assert ('Option "--checksumalgo" (%s) differs from the algorithm of the checksum list (%s)'
            % (given, listed)) in res.stderr, res.stderr


@pytest.mark.parametrize("chunk", [[], ["--checksumchunk", "64k"]])
def test_blake3_is_accepted(tmp_path, chunk):
    res = run_cli("--dryrun", *CLI, "--checksums", str(tmp_path / "sums"), "--checksumalgo",
                  "blake3", *chunk, str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr


def test_unknown_name_names_blake3(tmp_path):
    res = run_cli(*CLI, "--checksums", str(tmp_path / "s"), "--checksumalgo", "sha256",
                  str(tmp_path / "x"))
    assert res.returncode == 1
    assert 'Option "--checksumalgo" must be crc32, crc32c or crc64nvme, or blake3' in res.stderr


def test_help_text_names_blake3():
    res = run_cli("--help-all")
    text = " ".join(res.stdout.split())
    assert ("crc32 (zlib, gzip, zip), crc32c (Castagnoli: iSCSI, GCS, btrfs) or crc64nvme (NVMe "
            "protection information, S3), or blake3 (BLAKE3-256 as b3sum prints it, 64 hex "
            "digits; block size a multiple of 1K).") in text
    assert "Requires --checksums or --checksumverify. (Default: crc32)" in text


@pytest.mark.parametrize("block,size,unaligned,message", [
    (1536, 3 * MiB, False, 'Option "--checksumalgo" blake3 requires a block size that is a '
                           'multiple of 1K'),
    (MiB, 4 * MiB, True, 'Option "--checksumalgo" blake3 cannot be used together with '
                         '"--norandalign"'),
])
def test_config_rejections(tmp_path, block, size, unaligned, message):
    cfg = WorkerConfig(paths=[str(tmp_path / "f")], block_size=block, file_size=size,
                       checksums=not unaligned, checksum_algo="blake3",
                       use_random_offsets=unaligned, use_random_unaligned=unaligned)
    with pytest.raises(WorkerError) as excinfo:
        WorkerManager(cfg)
    assert str(excinfo.value) == message


def test_config_still_rejects_unknown_names(tmp_path):
    cfg = WorkerConfig(paths=[str(tmp_path / "f")], block_size=MiB, file_size=MiB,
                       checksums=True, checksum_algo="md5")
    with pytest.raises(WorkerError, match="^Invalid checksum algorithm: -1$"):
        WorkerManager(cfg)
