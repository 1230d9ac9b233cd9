"""CPU tests of --cdcreducestats: the model (N, D, B, U as --cdcstats counts them, S at most U and U
on random data, the shifted copy that only content-defined chunks deduplicate), the command line's
rejections, help text and dry run, the setter's and kernel entries' argument checks (without a
launch), and the console line."""
import ctypes

import pytest

from elbencho_b200 import _native, kernels
from tests import cdc_model, reduce_model
from tests import cdc_reduce_model as model
from tests.test_cli import run_cli
from tests.test_compress_stats import make_data

KiB, MiB = 1 << 10, 1 << 20
CLI = ["-w", "-r", "-b", "1m", "-s", "4m", "--gpuids", "0"]
RANGE = 'Option "--cdcreducestats" must be a power of two from 4K to 256K'


@pytest.mark.parametrize("avg", [4 * KiB, 16 * KiB, 64 * KiB])
@pytest.mark.parametrize("kind", ["random", "zero", "text", "blockvar"])
def test_model_counts_are_those_of_cdcstats(avg, kind):
    datas = [make_data(kind, MiB + 77, avg), make_data(kind, 512 * KiB, avg + 1)]
    n, d, b, u, s = model.counts(datas, 256 * KiB, avg)
    assert (n, d, b, u) == cdc_model.counts(datas, 256 * KiB, avg)
    assert s <= u
    if kind == "random":
        assert s == u
    else:
        assert s < u


def test_model_stores_each_distinct_chunk_once():
    data = make_data("blockvar", 2 * MiB, 3)
    one = model.counts([data], MiB, 16 * KiB)
    two = model.counts([data, data], MiB, 16 * KiB)
    assert two == (2 * one[0], one[1], 2 * one[2], one[3], one[4])


def test_shifted_copy():
    """--blockvarpct 50 data, 3 bytes, the data again: CDC dedupes about 2:1 where fixed 16K
    chunks find nothing, and the distinct chunks compress as the data does"""
    data = make_data("blockvar", 4 * MiB, 8)
    shifted = b"xyz" + data
    n, d, b, u, s = model.counts([data, shifted], MiB, 16 * KiB)
    assert b == 8 * MiB + 3 and 1.9 < b / u < 2.0
    assert 1.5 < u / s < 2.5
    fixed = reduce_model.counts([data, shifted], 16 * KiB)
    assert reduce_model.ratio(fixed[2], fixed[3]) == "1.00"


@pytest.mark.parametrize("size", ["4k", "16k", "256k"])
def test_cli_accepts(tmp_path, size):
    res = run_cli("--dryrun", *CLI, "--cdcreducestats", size, str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr
    assert "CDC reduce:" not in res.stdout


@pytest.mark.parametrize("extra", [["--cdcstats", "16k"], ["--cdcstats", "4k"],
                                   ["--reducestats", "16k"], ["--compressstats", "16k"]])
def test_cli_accepts_with(tmp_path, extra):
    res = run_cli("--dryrun", *CLI, "--cdcreducestats", "16k", *extra, str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr


@pytest.mark.parametrize("extra,message", [
    (["--cdcreducestats", "3k"], RANGE),
    (["--cdcreducestats", "2k"], RANGE),
    (["--cdcreducestats", "512k", "-b", "2m"], RANGE),
    (["--cdcreducestats", "256k", "-b", "512k"],
     'The block size (524288) must be at least the largest chunk of "--cdcreducestats" '
     '(1048576)'),
    (["--cdcreducestats", "16k", "--rand", "--norandalign"],
     'Option "--cdcreducestats" cannot be used together with "--norandalign"'),
    (["--cdcreducestats", "16k", "--rand"],
     'Option "--cdcreducestats" cannot be used together with "--rand"'),
    (["--cdcreducestats", "16k", "--infloop"],
     'Option "--cdcreducestats" cannot be used together with "--infloop"'),
    (["--cdcreducestats", "16k", "--rwmixpct", "50"],
     'Option "--cdcreducestats" cannot be used together with "--rwmixpct"'),
    (["--cdcreducestats", "16k", "--rwmixthr", "1"],
     'Option "--cdcreducestats" cannot be used together with "--rwmixthr"'),
    (["--cdcreducestats", "16k", "--hosts", "localhost"],
     'Option "--cdcreducestats" cannot be used together with "--hosts"'),
])
def test_cli_rejections(tmp_path, extra, message):
    res = run_cli(*CLI, *extra, str(tmp_path / "data"))
    assert res.returncode == 1
    assert message in res.stderr, res.stderr


def test_block_is_taken_after_the_file_size(tmp_path):
    res = run_cli("-w", "-b", "1m", "-s", "32k", "--gpuids", "0", "--cdcreducestats", "16k",
                  str(tmp_path / "data"))
    assert res.returncode == 1
    assert ('The block size (32768) must be at least the largest chunk of "--cdcreducestats" '
            '(65536)' in res.stderr)
    res = run_cli("--dryrun", "-w", "-b", "1m", "-s", "64k", "--gpuids", "0",
                  "--cdcreducestats", "16k", str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr


def test_help_text():
    text = " ".join(run_cli("--help-all").stdout.split())
    assert "--cdcreducestats arg" in text
    assert ('prints "CDC reduce: <N> chunks of <MIN> to <MAX> bytes, mean <B/N>, <D> distinct: <B> '
            'bytes, <U> distinct bytes stored as <S>: dedupe <B/U>:1, compress <U/S>:1, total '
            '<B/S>:1"') in text
    assert ("Cannot be used with --rand, --norandalign, --infloop, --rwmixpct, --rwmixthr or "
            "--hosts. [b200]") in text


def test_setter_and_stats_need_a_manager():
    lib = _native.load()
    out = [ctypes.c_uint64(7) for _ in range(5)]
    assert lib.elb_mgr_set_cdc_reduce_stats(None, 14) == -1
    assert _native.last_error() == "elb_mgr_set_cdc_reduce_stats: NULL manager"
    assert lib.elb_mgr_cdc_reduce_stats(None, *[ctypes.byref(v) for v in out]) == -1
    assert _native.last_error() == "elb_mgr_cdc_reduce_stats: NULL argument"


def test_kernel_entry_argument_checks():
    lib = _native.load()
    raw = kernels.pack_block_descs([(0x1000, 64 * KiB, 0, 0)])
    descs = ctypes.create_string_buffer(raw, len(raw))
    buf = ctypes.create_string_buffer(4096)  # (never reached by a launch: every call fails)
    launches = kernels.num_kernel_launches()

    insert = lib.elb_cdc_hash_insert_marks
    for shift in (11, 19):
        assert insert(descs, 1, shift, 64, buf, buf, None, buf, buf, 1024, buf, buf, None) == -1
        assert _native.last_error() == ("elb_cdc_hash_insert_marks: mean chunk shift %d is not in "
                                        "[12, 18]" % shift)
        assert lib.elb_cdc_lz4(descs, 1, shift, 64, buf, buf, buf, buf, None) == -1
        assert _native.last_error() == "elb_cdc_lz4: mean chunk shift %d is not in [12, 18]" % shift
    assert insert(descs, 1, 12, 64, buf, buf, None, buf, buf, 1000, buf, buf, None) == -1
    assert _native.last_error() == ("elb_cdc_hash_insert_marks: table size 1000 is not a power of "
                                    "two")
    assert insert(descs, 1, 12, 64, buf, buf, None, None, buf, 1024, buf, buf, None) == -1
    assert _native.last_error() == "elb_cdc_hash_insert_marks: NULL table or counters"
    for args in [(descs, 1, 12, 64, buf, buf, None, buf, buf, 1024, buf, None, None),
                 (descs, 1, 12, 64, buf, None, None, buf, buf, 1024, buf, buf, None),
                 (descs, 1, 12, 64, buf, buf, None, buf, None, 1024, buf, buf, None)]:
        assert insert(*args) == -1
        assert _native.last_error() == ("elb_cdc_hash_insert_marks: NULL payloads, descriptor, "
                                        "count, end or mark array")
    assert insert(descs, 1, 14, 15, buf, buf, None, buf, buf, 1024, buf, buf, None) == -1
    assert _native.last_error() == ("elb_cdc_hash_insert_marks: descriptor 0 can have 16 chunks, "
                                    "more than 15 slots per descriptor")
    for i in range(4, 8):
        args = [descs, 1, 12, 64, buf, buf, buf, buf, None]
        args[i] = None
        assert lib.elb_cdc_lz4(*args) == -1
        assert _native.last_error() == ("elb_cdc_lz4: NULL descriptor, count, end, mark or payload "
                                        "array")
    assert lib.elb_cdc_lz4(None, 1, 12, 64, buf, buf, buf, buf, None) == -1
    assert lib.elb_cdc_lz4(descs, 1, 12, 63, buf, buf, buf, buf, None) == -1
    assert _native.last_error() == ("elb_cdc_lz4: descriptor 0 can have 64 chunks, more than 63 "
                                    "slots per descriptor")
    # nothing to hash or compress: no launch
    assert insert(None, 0, 12, 64, None, None, None, buf, buf, 1024, buf, None, None) == 0
    assert lib.elb_cdc_lz4(None, 0, 12, 64, None, None, None, None, None) == 0
    assert kernels.num_kernel_launches() == launches


@pytest.mark.parametrize("avg,counts,line", [
    (16 * KiB, (0, 0, 0, 0, 0),
     "CDC reduce: 0 chunks of 4096 to 65536 bytes, mean 0, 0 distinct: 0 bytes, 0 distinct bytes "
     "stored as 0: dedupe 1.00:1, compress 1.00:1, total 1.00:1"),
    (16 * KiB, (453, 235, 8388611, 4285825, 2142000),
     "CDC reduce: 453 chunks of 4096 to 65536 bytes, mean 18517, 235 distinct: 8388611 bytes, "
     "4285825 distinct bytes stored as 2142000: dedupe 1.96:1, compress 2.00:1, total 3.92:1"),
    (4 * KiB, (64, 1, MiB, 16 * KiB, 77),
     "CDC reduce: 64 chunks of 1024 to 16384 bytes, mean 16384, 1 distinct: 1048576 bytes, 16384 "
     "distinct bytes stored as 77: dedupe 64.00:1, compress 212.78:1, total 13617.87:1"),
])
def test_console_line(avg, counts, line):
    assert kernels.cdc_reduce_line(avg, *counts) == line == model.line(avg, *counts)


def test_console_line_needs_counters():
    lib = _native.load()
    assert lib.elb_format_cdc_reduce_line(16 * KiB, None, None, 0) == -1
    assert _native.last_error() == "elb_format_cdc_reduce_line: NULL counters"
