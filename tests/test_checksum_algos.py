"""CPU tests of --checksumalgo: the generic model (tests/crc_algo_model.py) against zlib and the
published vectors of CRC-32C and CRC-64/NVME; the library's shift and finish of all three algorithms
against the model, for shifts past 2^31, 2^32 and near 2^64 and for random splits merged by XOR;
the list parser's headers, widths and errors; the command line and config rejections, the help
texts, the elb_cfg field and the argument checks of the new C ABI entries."""
import ctypes
import random
import zlib

import pytest

from elbencho_b200 import WorkerConfig, WorkerError, WorkerManager, _native, kernels
from tests import crc_algo_model as model
from tests.crc_model import random_split
from tests.test_cli import run_cli

KiB, MiB = 1 << 10, 1 << 20

ALGOS = list(model.ALGOS)
CLI = ["-r", "-b", "256k", "-s", "4m", "--gpuids", "0"]


# ------------------------------------------------------------------------------------------------
# the model
# ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("size", [0, 1, 7, 100, 4096, 10000])
def test_model_crc32_is_zlib(size):
    data = random.Random(size).randbytes(size)
    assert model.crc(model.ALGOS["crc32"], data) == zlib.crc32(data)


@pytest.mark.parametrize("algo,check", [
    ("crc32", 0xCBF43926), ("crc32c", 0xE3069283), ("crc64nvme", 0xAE8B14860A799888)])
def test_model_check_values(algo, check):
    assert model.crc(model.ALGOS[algo], b"123456789") == check


@pytest.mark.parametrize("data,want", [
    (bytes(32), 0x8A9136AA), (b"\xff" * 32, 0x62A8AB43), (bytes(range(32)), 0x46DD794E),
    (bytes(range(31, -1, -1)), 0x113FDB5C)])
def test_model_crc32c_rfc3720_vectors(data, want):
    assert model.crc(model.ALGOS["crc32c"], data) == want


@pytest.mark.parametrize("data,want", [
    (bytes(4096), 0x6482D367EB22B64E), (b"\xff" * 4096, 0xC0DDBA7302ECA3AC),
    (bytes(i & 0xFF for i in range(4096)), 0x3E729F5F6750449C)])
def test_model_crc64nvme_vectors(data, want):
    assert model.crc(model.ALGOS["crc64nvme"], data) == want


@pytest.mark.parametrize("algo", ALGOS)
def test_model_order_of_x(algo):
    a = model.ALGOS[algo]
    assert model._xpow(a, model.order_of_x(a)) == 1


# ------------------------------------------------------------------------------------------------
# the library's host arithmetic
# ------------------------------------------------------------------------------------------------

SHIFTS = [0, 1, 7, 4096, (1 << 31) - 2, (1 << 31) - 1, 1 << 31, 3 << 30, (1 << 32) - 1, 1 << 32,
          (1 << 32) + 5, 1 << 40, (1 << 63) + 12345, (1 << 64) - 2, (1 << 64) - 1]


@pytest.mark.parametrize("algo", ALGOS)
def test_library_shift_is_the_model(algo):
    a = model.ALGOS[algo]
    rng = random.Random(algo)
    for n in SHIFTS:
        crc = rng.getrandbits(a.width)
        assert kernels.crc_shift(crc, n, algo=algo) == model.shift(a, crc, n), n


@pytest.mark.parametrize("algo", ALGOS)
def test_library_finish_is_the_model(algo):
    a = model.ALGOS[algo]
    for size in [0, 1, 9, 4096, 65537]:
        data = random.Random(size).randbytes(size)
        raw = model.raw_crc(a, data)
        assert kernels.crc_finish(raw, size, algo=algo) == model.crc(a, data)
    for size in SHIFTS:  # (sizes no message of the tests could have)
        raw = random.Random(size).getrandbits(a.width)
        assert kernels.crc_finish(raw, size, algo=algo) == model.finish(a, raw, size), size


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("seed", range(4))
def test_random_splits_merge_by_xor(algo, seed):
    a = model.ALGOS[algo]
    rng = random.Random(seed)
    data = rng.randbytes(rng.choice([0, 1, 333, 5000]))
    raw = 0
    for offset, length in random_split(len(data), rng):
        part = model.raw_crc(a, data[offset:offset + length])
        raw ^= kernels.crc_shift(part, len(data) - offset - length, algo=algo)
    assert raw == model.raw_crc(a, data)
    assert kernels.crc_finish(raw, len(data), algo=algo) == model.crc(a, data)


def test_crc32_entries_are_the_crc32_case():
    rng = random.Random(3)
    for n in SHIFTS:
        crc = rng.getrandbits(32)
        assert kernels.crc32_shift(crc, n) == kernels.crc_shift(crc, n, algo="crc32")
        assert kernels.crc32_finish(crc, n) == kernels.crc_finish(crc, n, algo="crc32")


def test_crc32c_is_reduced_by_its_own_order():
    """x^(2^31 - 1) = 1 for CRC-32C: a shift by the order is the identity, one by 2^32 - 1 is not"""
    crc = 0x12345678
    assert kernels.crc_shift(crc, (1 << 31) - 1, algo="crc32c") == model.shift(
        model.ALGOS["crc32c"], crc, 0) == crc
    assert kernels.crc_shift(crc, (1 << 32) - 1, algo="crc32c") != crc


# ------------------------------------------------------------------------------------------------
# the C ABI
# ------------------------------------------------------------------------------------------------

def test_crc_chunks_argument_checks():
    lib = _native.load()
    raw = kernels.pack_block_descs([(0x1000, 16, 0, 0)])
    descs = ctypes.create_string_buffer(raw, len(raw))
    crcs = (ctypes.c_uint64 * 4)(0)
    for algo in (-1, 3):
        assert lib.elb_crc_chunks(algo, descs, None, 1, 12, 1, crcs, None, None, None) == -1
        assert _native.last_error() == "elb_crc_chunks: unknown checksum algorithm %d" % algo
    assert lib.elb_crc_chunks(2, descs, None, 1, 11, 1, crcs, None, None, None) == -1
    assert _native.last_error() == "elb_crc_chunks: chunk shift 11 is neither 64 nor in [12, 40]"
    assert lib.elb_crc_chunks(1, descs, None, 1, 12, 0, crcs, None, None, None) == -1
    assert "elb_crc_chunks: slots per descriptor must be at least 1" in _native.last_error()
    assert lib.elb_crc_chunks(2, descs, None, 1, 64, 1, crcs, None, None, None) == -1
    assert _native.last_error() == "elb_crc_chunks: NULL descriptor, shift or CRC array"
    assert lib.elb_crc_chunks(1, descs, None, 1, 12, 1, crcs, crcs, None, None) == -1
    assert _native.last_error() == "elb_crc_chunks: host CRCs and device ticket go together"
    raw = kernels.pack_block_descs([(0x1000, 8192, 4095, 0)])
    descs = ctypes.create_string_buffer(raw, len(raw))
    assert lib.elb_crc_chunks(2, descs, None, 1, 12, 2, crcs, None, None, None) == -1
    assert "descriptor 0 spans 3 chunks, more than 2 slots" in _native.last_error()
    assert lib.elb_crc_chunks(2, None, None, 0, 12, 1, None, None, None, None) == 0
    with pytest.raises(kernels.KernelError, match="unknown checksum algorithm 'md5'"):
        kernels.crc_chunks(0, 0, 0, 12, 1, 0, algo="md5")


@pytest.mark.parametrize("entry", ["elb_crc_shift", "elb_crc_finish"])
def test_crc_shift_and_finish_reject_unknown_algorithms(entry):
    lib = _native.load()
    assert getattr(lib, entry)(3, 0x1234, 5) == 0
    assert _native.last_error() == "%s: unknown checksum algorithm 3" % entry
    assert getattr(lib, entry)(2, 0x1234, 5) != 0


def test_cfg_field_fills_padding():
    assert ctypes.sizeof(_native.Cfg) == _native.load().elb_cfg_struct_size() == 360
    assert _native.Cfg.useStridedAccess.offset == 120
    assert _native.Cfg.checksumAlgo.offset == 124
    assert _native.Cfg.randomAmount.offset == 128


def test_config_rejects_unknown_algorithm(tmp_path):
    cfg = WorkerConfig(paths=[str(tmp_path / "f")], block_size=MiB, file_size=MiB,
                       checksums=True, checksum_algo="md5")
    with pytest.raises(WorkerError) as excinfo:
        WorkerManager(cfg)
    assert str(excinfo.value) == "Invalid checksum algorithm: -1"


# ------------------------------------------------------------------------------------------------
# the list parser (the library's, through the command line's dry run)
# ------------------------------------------------------------------------------------------------

def dry_run(tmp_path, text, *extra):
    lst = tmp_path / "list"
    lst.write_text(text)
    return run_cli("--dryrun", *CLI, *extra, "--checksumverify", str(lst), str(tmp_path / "data"))


@pytest.mark.parametrize("text", [
    "# phase WRITE chunk 65536 crc32c\n/a 0 65536 0000abcd\n",
    "# phase READ chunk 4096 crc64nvme\n/a 0 4096 0123456789ABCDEF\n/a 4096 7 fedcba9876543210\n",
    "# phase WRITE chunk 4096 crc32\n/a 0 4096 00000000\n",
    "# phase WRITE crc64nvme\n/a 4096 4096 0123456789abcdef\n# phase WRITE crc32c\n/a 1 1 -\n"
    "# phase READ chunk 65536 crc32c\n/a 0 65536 0000abcd\n",
])
def test_lists_of_every_algorithm_parse(tmp_path, text):
    res = dry_run(tmp_path, text)
    assert res.returncode == 0, res.stderr


@pytest.mark.parametrize("text,line_num,reason", [
    ("# phase WRITE chunk 65536 crc64nvme\n/a 0 65536 0000abcd\n", 2,
     'not "path offset length crc64nvme"'),
    ("# phase WRITE chunk 65536 crc64nvme\n/a 0 65536 00000000000000000\n", 2,
     'not "path offset length crc64nvme"'),
    ("# phase WRITE chunk 65536 crc32c\n\n/a 0 65536 0123456789abcdef\n", 3,
     'not "path offset length crc32c"'),
    ("# phase WRITE chunk 65536\n/a 0 65536 0123456789abcdef\n", 2,
     'not "path offset length crc32"'),
    ("# phase WRITE chunk 65536 crc16\n", 1, "not a phase header"),
    ("# phase WRITE chunk 65536 crc32c x\n", 1, "not a phase header"),
    ("# phase WRITE md5\n", 1, "not a phase header"),
])
def test_malformed_lines_name_their_line(tmp_path, text, line_num, reason):
    res = dry_run(tmp_path, text)
    assert res.returncode == 1
    assert "Checksum list line %d: %s: " % (line_num, reason) in res.stderr, res.stderr


@pytest.mark.parametrize("given,listed", [
    ("crc32", "crc32c"), ("crc64nvme", "crc32c"), ("crc32c", "crc32")])
def test_explicit_algorithm_must_match_the_list(tmp_path, given, listed):
    header = "# phase WRITE chunk 65536" + ("" if listed == "crc32" else " " + listed)
    res = dry_run(tmp_path, header + "\n/a 0 65536 0000abcd\n", "--checksumalgo", given)
    assert res.returncode == 1
    assert ('Option "--checksumalgo" (%s) differs from the algorithm of the checksum list (%s)'
            % (given, listed)) in res.stderr, res.stderr
    res = dry_run(tmp_path, header + "\n/a 0 65536 0000abcd\n", "--checksumalgo", listed)
    assert res.returncode == 0, res.stderr


# ------------------------------------------------------------------------------------------------
# command line
# ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("extra,message", [
    ([], 'Option "--checksumalgo" requires "--checksums" or "--checksumverify"'),
    (["--checksums", "/tmp/elb_sums", "--checksumalgo", "crc16"],
     'Option "--checksumalgo" must be crc32, crc32c or crc64nvme'),
    (["--checksums", "/tmp/elb_sums", "--hosts", "localhost:1"],
     'Option "--checksums" cannot be used together with "--hosts"'),
])
def test_validation_messages(tmp_path, extra, message):
    res = run_cli(*CLI, "--checksumalgo", "crc32c", *extra, str(tmp_path / "x"))
    assert res.returncode == 1
    assert message in res.stderr, res.stderr


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("chunk", [[], ["--checksumchunk", "64k"]])
def test_accepted_combinations(tmp_path, algo, chunk):
    res = run_cli("--dryrun", *CLI, "--checksums", str(tmp_path / "sums"), "--checksumalgo", algo,
                  *chunk, str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr


def test_help_texts():
    res = run_cli("--help-all")
    assert res.returncode == 0
    text = " ".join(res.stdout.split())
    assert "--checksumalgo" in text
    assert ("crc32 (zlib, gzip, zip), crc32c (Castagnoli: iSCSI, GCS, btrfs) or crc64nvme (NVMe "
            "protection information, S3)") in text
    assert "Requires --checksums or --checksumverify. (Default: crc32)" in text
    assert "computes the CRC (--checksumalgo) of each file" in text
    assert 'one line "path size bytes_covered crc" per file' in text
    assert 'lists the CRC of every chunk the phase moved' in text
    assert "every read phase checks the CRC of each chunk it reads" in text
    assert "CRC-32" not in text
