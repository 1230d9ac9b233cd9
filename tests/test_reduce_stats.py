"""CPU tests of --reducestats: the model's counts on hand-built data, the command line's rejections,
help text and dry run, the setter's and kernel entries' argument checks, and the console line."""
import ctypes

import pytest

from elbencho_b200 import _native, kernels
from tests import compress_model, reduce_model as model
from tests.test_cli import run_cli
from tests.test_compress_stats import make_data

KiB, MiB = 1 << 10, 1 << 20

CLI = ["-w", "-r", "-b", "256k", "-s", "4m", "--gpuids", "0"]


def test_model_all_zeros():
    data = bytes(256 * KiB)
    assert model.counts([data], 64 * KiB) == (4, 1, 256 * KiB, 64 * KiB, 267)


def test_model_all_distinct():
    data = make_data("random", 256 * KiB, 1)
    n, d, b, u, s = model.counts([data], 64 * KiB)
    assert (n, d, b, u) == (4, 4, 256 * KiB, 256 * KiB)
    assert s == 256 * KiB  # (random chunks do not shrink: each is stored at its length)


def test_model_one_chunk_repeated():
    chunk = make_data("text", 4 * KiB, 2)
    other = make_data("random", 4 * KiB, 3)
    n, d, b, u, s = model.counts([chunk * 5 + other, chunk], 4 * KiB)
    assert (n, d, b, u) == (7, 2, 28 * KiB, 8 * KiB)
    assert s == compress_model.size(chunk) + 4 * KiB


def test_model_short_last_chunks():
    # a short last chunk is a chunk of its own length; the same bytes at the same length are one
    tail = make_data("acgt", 1000, 4)
    full = bytes(4 * KiB)
    n, d, b, u, s = model.counts([full + tail, full + tail, tail], 4 * KiB)
    assert (n, d, b, u) == (5, 2, 2 * (4 * KiB + 1000) + 1000, 4 * KiB + 1000)
    assert s == compress_model.size(full) + min(compress_model.size(tail), 1000)
    # a zero chunk and a short zero chunk differ
    assert model.counts([bytes(4 * KiB + 100)], 4 * KiB)[1] == 2


def test_model_totals_are_products():
    datas = [make_data("blockvar", 64 * KiB, 5) * 3, bytes(64 * KiB)]
    n, d, b, u, s = model.counts(datas, 16 * KiB)
    assert n == 16 and b == 256 * KiB and d < n
    dedupe, compress, total = (float(x) for x in model.line(16 * KiB, n, d, b, u, s)
                               .split("dedupe ")[1].replace(":1", "")
                               .replace("compress ", "").replace("total ", "").split(", "))
    assert abs(dedupe * compress - total) < 0.01 * total + 0.01


@pytest.mark.parametrize("size", ["4k", "64k", "256k"])
def test_cli_accepts(tmp_path, size):
    res = run_cli("--dryrun", *CLI, "--reducestats", size, str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr


@pytest.mark.parametrize("extra", [["--dedupestats", "64k"], ["--dedupestats", "4k"],
                                   ["--compressstats", "64k"], ["--compressstats", "16k"],
                                   ["--checksums", "--checksumalgo", "blake3",
                                    "--checksumchunk", "64k"]])
def test_cli_accepts_with(tmp_path, extra):
    if "--checksums" in extra:
        extra = [extra[0], str(tmp_path / "sums")] + extra[1:]
    res = run_cli("--dryrun", *CLI, "--reducestats", "64k", *extra, str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr


@pytest.mark.parametrize("extra,message", [
    (["--reducestats", "3k"], 'Option "--reducestats" must be a power of two from 4K to 1M'),
    (["--reducestats", "2k"], 'Option "--reducestats" must be a power of two from 4K to 1M'),
    (["--reducestats", "2m"], 'Option "--reducestats" must be a power of two from 4K to 1M'),
    (["--reducestats", "1m"], 'The block size (262144) must be a multiple of "--reducestats" '
                              '(1048576)'),
    (["--reducestats", "64k", "--rand", "--norandalign"],
     'Option "--reducestats" cannot be used together with "--norandalign"'),
    (["--reducestats", "64k", "--rand"],
     'Option "--reducestats" cannot be used together with "--rand"'),
    (["--reducestats", "64k", "--infloop"],
     'Option "--reducestats" cannot be used together with "--infloop"'),
    (["--reducestats", "64k", "--rwmixpct", "50"],
     'Option "--reducestats" cannot be used together with "--rwmixpct"'),
    (["--reducestats", "64k", "--rwmixthr", "1"],
     'Option "--reducestats" cannot be used together with "--rwmixthr"'),
    (["--reducestats", "64k", "--hosts", "localhost"],
     'Option "--reducestats" cannot be used together with "--hosts"'),
])
def test_cli_rejections(tmp_path, extra, message):
    res = run_cli(*CLI, *extra, str(tmp_path / "data"))
    assert res.returncode == 1
    assert message in res.stderr, res.stderr


def test_block_reduced_to_the_file_size_is_accepted(tmp_path):
    res = run_cli("--dryrun", "-w", "-b", "1m", "-s", "100k", "--gpuids", "0", "--reducestats",
                  "64k", str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr


def test_block_smaller_than_the_file_is_checked(tmp_path):
    res = run_cli("-w", "-b", "96k", "-s", "200k", "--gpuids", "0", "--reducestats", "64k",
                  str(tmp_path / "data"))
    assert res.returncode == 1
    assert 'The block size (98304) must be a multiple of "--reducestats" (65536)' in res.stderr


def test_dry_run_prints_no_line(tmp_path):
    res = run_cli("--dryrun", *CLI, "--reducestats", "64k", str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr
    assert "Reduce:" not in res.stdout


def test_help_text():
    text = " ".join(run_cli("--help-all").stdout.split())
    assert "--reducestats arg" in text
    assert ('It prints "Reduce: <N> chunks of <K>, <D> distinct: <B> bytes, <U> distinct bytes '
            'stored as <S>: dedupe <B/U>:1, compress <U/S>:1, total <B/S>:1"') in text
    assert ("Cannot be used with --rand, --norandalign, --infloop, --rwmixpct, --rwmixthr or "
            "--hosts. [b200]") in text


def test_setter_and_stats_need_a_manager():
    lib = _native.load()
    out = [ctypes.c_uint64(7) for _ in range(5)]
    assert lib.elb_mgr_set_reduce_stats(None, 16) == -1
    assert _native.last_error() == "elb_mgr_set_reduce_stats: NULL manager"
    assert lib.elb_mgr_reduce_stats(None, *[ctypes.byref(v) for v in out]) == -1
    assert _native.last_error() == "elb_mgr_reduce_stats: NULL argument"


def test_kernel_entry_argument_checks():
    lib = _native.load()
    raw = kernels.pack_block_descs([(0x1000, 64 * KiB, 0, 0)])
    descs = ctypes.create_string_buffer(raw, len(raw))
    buf = ctypes.create_string_buffer(4096)  # (never reached by a launch: every call fails)

    assert lib.elb_reduce_insert(descs, 1, 12, 16, buf, buf, 1000, buf, buf, None) == -1
    assert _native.last_error() == "elb_reduce_insert: table size 1000 is not a power of two"
    assert lib.elb_reduce_insert(descs, 1, 12, 16, buf, None, 1024, buf, buf, None) == -1
    assert _native.last_error() == "elb_reduce_insert: NULL table or counters"
    assert lib.elb_reduce_insert(descs, 1, 12, 16, buf, buf, 1024, buf, None, None) == -1
    assert _native.last_error() == "elb_reduce_insert: NULL descriptor, digest or mark array"
    for shift in (11, 21):
        assert lib.elb_reduce_insert(descs, 1, shift, 16, buf, buf, 1024, buf, buf, None) == -1
        assert _native.last_error() == ("elb_reduce_insert: chunk shift %d is not in [12, 20]"
                                        % shift)
        assert lib.elb_reduce_lz4(descs, 1, shift, 16, buf, buf, None) == -1
        assert _native.last_error() == "elb_reduce_lz4: chunk shift %d is not in [12, 20]" % shift
    assert lib.elb_reduce_lz4(descs, 1, 12, 16, buf, None, None) == -1
    assert _native.last_error() == "elb_reduce_lz4: NULL descriptor, mark or payload array"
    off = kernels.pack_block_descs([(0x1000, 64 * KiB, 2 * KiB, 0)])
    off_descs = ctypes.create_string_buffer(off, len(off))
    assert lib.elb_reduce_lz4(off_descs, 1, 12, 16, buf, buf, None) == -1
    assert _native.last_error() == ("elb_reduce_lz4: descriptor 0 (offset 2048) is not on a chunk "
                                    "boundary")
    assert lib.elb_reduce_insert(descs, 1, 12, 15, buf, buf, 1024, buf, buf, None) == -1
    assert _native.last_error() == ("elb_reduce_insert: descriptor 0 has 16 chunks, more than 15 "
                                    "slots per descriptor")
    assert lib.elb_reduce_merge(buf, None, 5, buf, buf, 1024, buf, None) == -1
    assert _native.last_error() == "elb_reduce_merge: NULL payloads or source entries"
    assert lib.elb_reduce_merge(buf, buf, 5, buf, buf, 3, buf, None) == -1
    assert _native.last_error() == "elb_reduce_merge: table size 3 is not a power of two"
    assert lib.elb_reduce_sum(buf, None, 1024, buf, None) == -1
    assert _native.last_error() == "elb_reduce_sum: NULL payloads"
    assert lib.elb_reduce_sum(buf, buf, 1024, None, None) == -1
    assert _native.last_error() == "elb_reduce_sum: NULL table or counters"
    # nothing to insert, compress or merge: no launch
    assert lib.elb_reduce_insert(None, 0, 12, 16, None, buf, 1024, buf, None, None) == 0
    assert lib.elb_reduce_lz4(None, 0, 12, 16, None, None, None) == 0
    assert lib.elb_reduce_merge(None, None, 0, buf, buf, 1024, buf, None) == 0


@pytest.mark.parametrize("counts,line", [
    ((0, 0, 0, 0, 0), "Reduce: 0 chunks of 65536, 0 distinct: 0 bytes, 0 distinct bytes stored as "
                      "0: dedupe 1.00:1, compress 1.00:1, total 1.00:1"),
    ((16, 1, 1 << 20, 65536, 267),
     "Reduce: 16 chunks of 65536, 1 distinct: 1048576 bytes, 65536 distinct bytes stored as 267: "
     "dedupe 16.00:1, compress 245.45:1, total 3927.25:1"),
    ((4, 3, 262144, 196608, 98304),
     "Reduce: 4 chunks of 65536, 3 distinct: 262144 bytes, 196608 distinct bytes stored as 98304: "
     "dedupe 1.33:1, compress 2.00:1, total 2.67:1"),
])
def test_console_line(counts, line):
    n, d, b, u, s = counts
    assert kernels.reduce_line(64 * KiB, n, d, b, u, s) == line
    assert model.line(64 * KiB, n, d, b, u, s) == line
