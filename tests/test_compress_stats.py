"""CPU tests of --compressstats: the LZ4 parse model round-trips through the block decoder and keeps
the block rules, gives the worked sizes of DESIGN.md, the command line's rejections and help text,
the setter's NULL checks, the argument checks of elb_lz4_chunks and the console line."""
import ctypes

import numpy as np
import pytest

from elbencho_b200 import _native, kernels
from tests import compress_model as model
from tests.test_cli import run_cli

KiB, MiB = 1 << 10, 1 << 20

CLI = ["-w", "-r", "-b", "256k", "-s", "4m", "--gpuids", "0"]

LENGTHS = list(range(0, 14)) + [4 * KiB, 64 * KiB, 64 * KiB + 1, MiB]


def blockvar_data(n, pct, seed):
    """--blockvarpct style: pct percent of each 4 KiB random, the rest one repeated byte"""
    rng = np.random.default_rng(seed)
    out = np.full(n, rng.integers(0, 256), dtype=np.uint8)
    for o in range(0, n, 4 * KiB):
        k = min(4 * KiB, n - o) * pct // 100
        out[o:o + k] = rng.integers(0, 256, k, dtype=np.uint8)
    return out.tobytes()


def make_data(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "zero":
        return bytes(n)
    if kind == "random":
        return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    if kind == "acgt":
        return rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), n).tobytes()
    if kind == "text":
        words = [b"block", b"chunk", b"storage", b"ratio", b"the", b"of", b"gpu", b"lz4"]
        text = b" ".join(words[i] for i in rng.integers(0, len(words), n // 3 + 1))
        return text[:n]
    return blockvar_data(n, 50, seed)


@pytest.mark.parametrize("kind", ["zero", "random", "acgt", "text", "blockvar"])
@pytest.mark.parametrize("n", LENGTHS)
def test_model_round_trips(kind, n):
    if kind == "acgt" and n == MiB:
        n = 256 * KiB  # (the slowest data for the model in Python)
    data = make_data(kind, n, n + 7)
    block = model.compress(data)
    assert len(block) == model.size(data)
    assert model.decode(block) == data
    model.check_block_rules(data)
    if n < 13:
        assert block == bytes([min(n, 15) << 4]) + data


@pytest.mark.parametrize("data,size", [(bytes(4 * KiB), 26), (bytes(64 * KiB), 267),
                                       (None, 4114), (None, 65794)])
def test_worked_sizes(data, size):
    if data is None:
        data = make_data("random", 4 * KiB if size == 4114 else 64 * KiB, 3)
    assert model.size(data) == size


def test_decoder_rejects_a_bad_offset():
    with pytest.raises(ValueError):
        model.decode(bytes([0x10, 65, 5, 0, 0x00]))


@pytest.mark.parametrize("size", ["4k", "64k", "256k"])
def test_cli_accepts(tmp_path, size):
    res = run_cli("--dryrun", *CLI, "--compressstats", size, str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr


@pytest.mark.parametrize("extra", [["--rand"], ["--infloop"], ["--dedupestats", "64k"]])
def test_cli_accepts_with(tmp_path, extra):
    res = run_cli("--dryrun", *CLI, "--compressstats", "64k", *extra, str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr


@pytest.mark.parametrize("extra,message", [
    (["--compressstats", "3k"], 'Option "--compressstats" must be a power of two from 4K to 1M'),
    (["--compressstats", "2k"], 'Option "--compressstats" must be a power of two from 4K to 1M'),
    (["--compressstats", "2m"], 'Option "--compressstats" must be a power of two from 4K to 1M'),
    (["--compressstats", "1m"], 'The block size (262144) must be a multiple of "--compressstats" '
                                '(1048576)'),
    (["--compressstats", "64k", "--rand", "--norandalign"],
     'Option "--compressstats" cannot be used together with "--norandalign"'),
    (["--compressstats", "64k", "--rwmixpct", "50"],
     'Option "--compressstats" cannot be used together with "--rwmixpct"'),
    (["--compressstats", "64k", "--rwmixthr", "1"],
     'Option "--compressstats" cannot be used together with "--rwmixthr"'),
    (["--compressstats", "64k", "--hosts", "localhost"],
     'Option "--compressstats" cannot be used together with "--hosts"'),
])
def test_cli_rejections(tmp_path, extra, message):
    res = run_cli(*CLI, *extra, str(tmp_path / "data"))
    assert res.returncode == 1
    assert message in res.stderr, res.stderr


def test_block_reduced_to_the_file_size_is_accepted(tmp_path):
    res = run_cli("--dryrun", "-w", "-b", "1m", "-s", "100k", "--gpuids", "0", "--compressstats",
                  "64k", str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr


def test_help_text():
    text = " ".join(run_cli("--help-all").stdout.split())
    assert "--compressstats arg" in text
    assert ('prints "Compress: <N> chunks of <K>, <U> incompressible: <B> bytes to <S>: <B/S>:1", '
            "where S counts a chunk that does not shrink at its own length.") in text
    assert "Cannot be used with --norandalign, --rwmixpct, --rwmixthr or --hosts. [b200]" in text


def test_setter_and_stats_need_a_manager():
    lib = _native.load()
    out = [ctypes.c_uint64(7) for _ in range(4)]
    assert lib.elb_mgr_set_compress_stats(None, 12) == -1
    assert _native.last_error() == "elb_mgr_set_compress_stats: NULL manager"
    assert lib.elb_mgr_compress_stats(None, *[ctypes.byref(v) for v in out]) == -1
    assert _native.last_error() == "elb_mgr_compress_stats: NULL argument"


def test_lz4_chunks_argument_checks():
    lib = _native.load()
    raw = kernels.pack_block_descs([(0x1000, 64 * KiB, 0, 0)])
    descs = ctypes.create_string_buffer(raw, len(raw))
    buf = ctypes.create_string_buffer(4096)  # (never reached by a launch: every call fails)

    assert lib.elb_lz4_chunks(None, 1, 12, 16, buf, None, None, None) == -1
    assert _native.last_error() == "elb_lz4_chunks: NULL descriptor array or counters"
    assert lib.elb_lz4_chunks(descs, 1, 12, 16, None, None, None, None) == -1
    assert _native.last_error() == "elb_lz4_chunks: NULL descriptor array or counters"
    for shift in (11, 21, 64):
        assert lib.elb_lz4_chunks(descs, 1, shift, 16, buf, None, None, None) == -1
        assert _native.last_error() == "elb_lz4_chunks: chunk shift %d is not in [12, 20]" % shift
    off = kernels.pack_block_descs([(0x1000, 64 * KiB, 2 * KiB, 0)])
    off_descs = ctypes.create_string_buffer(off, len(off))
    assert lib.elb_lz4_chunks(off_descs, 1, 12, 16, buf, None, None, None) == -1
    assert _native.last_error() == ("elb_lz4_chunks: descriptor 0 (offset 2048) is not on a chunk "
                                    "boundary")
    assert lib.elb_lz4_chunks(descs, 1, 12, 15, buf, None, None, None) == -1
    assert _native.last_error() == ("elb_lz4_chunks: descriptor 0 has 16 chunks, more than 15 "
                                    "slots per descriptor")
    # nothing to compress: no launch
    assert lib.elb_lz4_chunks(None, 0, 12, 16, buf, None, None, None) == 0


@pytest.mark.parametrize("counts,line", [
    ((0, 0, 0, 0), "Compress: 0 chunks of 65536, 0 incompressible: 0 bytes to 0: 1.00:1"),
    ((16, 1 << 20, 4272, 0),
     "Compress: 16 chunks of 65536, 0 incompressible: 1048576 bytes to 4272: 245.45:1"),
    ((3, 139264, 139264, 3),
     "Compress: 3 chunks of 65536, 3 incompressible: 139264 bytes to 139264: 1.00:1"),
    ((5, 20000, 10001, 1), "Compress: 5 chunks of 65536, 1 incompressible: 20000 bytes to 10001: "
                           "2.00:1"),
])
def test_console_line(counts, line):
    assert kernels.compress_line(64 * KiB, *counts) == line


def test_counts_of_the_model():
    data = bytes(64 * KiB) + make_data("random", 64 * KiB + 100, 5)
    n, b, s, u = model.counts([data], 64 * KiB)
    assert (n, b, u) == (3, len(data), 2)
    assert s == 267 + 64 * KiB + 100
