"""CPU tests of --cdcstats: the model against the hash's definition and the gear table against
mix(), the chunk length bounds, cuts falling back in step after an insertion, the command line's
rejections, help text and dry run, the setter's and kernel entries' argument checks (without a
launch), and the console line."""
import ctypes

import numpy as np
import pytest

from elbencho_b200 import _native, kernels
from tests import cdc_model as model
from tests.test_cli import run_cli
from tests.test_compress_stats import make_data
from tests.verify_random_model import mix

KiB, MiB = 1 << 10, 1 << 20
CLI = ["-w", "-r", "-b", "1m", "-s", "4m", "--gpuids", "0"]


def test_gear_table():
    assert kernels.CDC_GEAR_TAG == model.GEAR_TAG == 0x6A09E667F3BCC908
    assert [int(g) for g in model.GEAR] == [mix(model.GEAR_TAG + i) for i in range(256)]


@pytest.mark.parametrize("kind", ["random", "zero", "text", "blockvar"])
def test_hash_doubling_is_the_definition(kind):
    block = make_data(kind, 3000, 17)
    h = model.hashes(block)
    for p in list(range(70)) + list(range(1000, 3000, 97)) + [2999]:
        assert int(h[p]) == model.hash_at(block, p), p


def test_cut_rule_by_hand():
    """strict before AVG, loose from AVG on, MAX if neither"""
    avg = 4 * KiB
    block = make_data("random", 64 * KiB, 3)
    h = model.hashes(block)
    strict, loose = h < np.uint64(1 << 50), h < np.uint64(1 << 54)
    c = 0
    for length in model.cut_lengths(block, avg):
        if c + 16 * KiB > len(block):
            break
        ls = [p - c + 1 for p in range(c + KiB - 1, c + avg - 1) if strict[p]]
        ll = [p - c + 1 for p in range(c + avg - 1, c + 16 * KiB - 1) if loose[p]]
        assert length == (ls[0] if ls else ll[0] if ll else 16 * KiB)
        c += length


@pytest.mark.parametrize("avg", [4 * KiB, 16 * KiB, 256 * KiB])
@pytest.mark.parametrize("kind", ["random", "zero", "text", "blockvar"])
def test_lengths_are_bounded(avg, kind):
    block = make_data(kind, 4 * MiB + 123, avg)
    lengths = model.cut_lengths(block, avg)
    assert sum(lengths) == len(block)
    assert all(avg // 4 <= n <= 4 * avg for n in lengths[:-1])
    assert 0 < lengths[-1] <= 4 * avg
    if kind == "random":
        assert 1.0 * avg < np.mean(lengths[:-1]) < 1.3 * avg


@pytest.mark.parametrize("avg", [4 * KiB, 16 * KiB, 64 * KiB])
def test_cuts_resynchronise_after_an_insertion(avg):
    data = make_data("random", 4 * MiB, avg + 1)
    shifted = data[:1000] + b"abc" + data[1000:]
    a = [off for off, _ in model.chunks(data, len(data), avg)]
    b = [off - 3 for off, _ in model.chunks(shifted, len(shifted), avg)]
    # past the first chunks both cut at the same content
    assert len(set(a) & set(b)) >= len(a) - 3
    n, d, total, u = model.counts([data, shifted], 4 * MiB + 3, avg)
    assert total == 2 * len(data) + 3 and total / u > 1.9


def test_counts_of_a_shifted_copy():
    data = make_data("random", 2 * MiB, 8)
    n, d, b, u = model.counts([data + b"xyz" + data], MiB, 16 * KiB)
    assert b == 4 * MiB + 3 and d < n and 1.8 < b / u < 2.0


@pytest.mark.parametrize("size", ["4k", "16k", "256k"])
def test_cli_accepts(tmp_path, size):
    res = run_cli("--dryrun", *CLI, "--cdcstats", size, str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr
    assert "CDC:" not in res.stdout


@pytest.mark.parametrize("extra", [["--dedupestats", "16k"], ["--reducestats", "64k"],
                                   ["--compressstats", "16k"]])
def test_cli_accepts_with(tmp_path, extra):
    res = run_cli("--dryrun", *CLI, "--cdcstats", "16k", *extra, str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr


@pytest.mark.parametrize("extra,message", [
    (["--cdcstats", "3k"], 'Option "--cdcstats" must be a power of two from 4K to 256K'),
    (["--cdcstats", "2k"], 'Option "--cdcstats" must be a power of two from 4K to 256K'),
    (["--cdcstats", "512k"], 'Option "--cdcstats" must be a power of two from 4K to 256K'),
    (["--cdcstats", "512k", "-b", "2m"],
     'Option "--cdcstats" must be a power of two from 4K to 256K'),
    (["--cdcstats", "256k", "-b", "512k"],
     'The block size (524288) must be at least the largest chunk of "--cdcstats" (1048576)'),
    (["--cdcstats", "16k", "--rand", "--norandalign"],
     'Option "--cdcstats" cannot be used together with "--norandalign"'),
    (["--cdcstats", "16k", "--rand"], 'Option "--cdcstats" cannot be used together with "--rand"'),
    (["--cdcstats", "16k", "--infloop"],
     'Option "--cdcstats" cannot be used together with "--infloop"'),
    (["--cdcstats", "16k", "--rwmixpct", "50"],
     'Option "--cdcstats" cannot be used together with "--rwmixpct"'),
    (["--cdcstats", "16k", "--rwmixthr", "1"],
     'Option "--cdcstats" cannot be used together with "--rwmixthr"'),
    (["--cdcstats", "16k", "--hosts", "localhost"],
     'Option "--cdcstats" cannot be used together with "--hosts"'),
])
def test_cli_rejections(tmp_path, extra, message):
    res = run_cli(*CLI, *extra, str(tmp_path / "data"))
    assert res.returncode == 1
    assert message in res.stderr, res.stderr


def test_block_is_taken_after_the_file_size(tmp_path):
    # a 1M block of a 32K file is a 32K block, below the 64K largest chunk
    res = run_cli("-w", "-b", "1m", "-s", "32k", "--gpuids", "0", "--cdcstats", "16k",
                  str(tmp_path / "data"))
    assert res.returncode == 1
    assert ('The block size (32768) must be at least the largest chunk of "--cdcstats" (65536)'
            in res.stderr)
    res = run_cli("--dryrun", "-w", "-b", "1m", "-s", "64k", "--gpuids", "0", "--cdcstats", "16k",
                  str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr


def test_help_text():
    text = " ".join(run_cli("--help-all").stdout.split())
    assert "--cdcstats arg" in text
    assert ('prints "CDC: <N> chunks of <MIN> to <MAX> bytes, mean <B/N>, <D> distinct: <B> bytes, '
            '<U> distinct bytes: <B/U>:1"') in text
    assert ("Cannot be used with --rand, --norandalign, --infloop, --rwmixpct, --rwmixthr or "
            "--hosts. [b200]") in text


def test_setter_and_stats_need_a_manager():
    lib = _native.load()
    out = [ctypes.c_uint64(7) for _ in range(4)]
    assert lib.elb_mgr_set_cdc_stats(None, 14) == -1
    assert _native.last_error() == "elb_mgr_set_cdc_stats: NULL manager"
    assert lib.elb_mgr_cdc_stats(None, *[ctypes.byref(v) for v in out]) == -1
    assert _native.last_error() == "elb_mgr_cdc_stats: NULL argument"


def test_kernel_entry_argument_checks():
    lib = _native.load()
    raw = kernels.pack_block_descs([(0x1000, 64 * KiB, 0, 0)])
    descs = ctypes.create_string_buffer(raw, len(raw))
    buf = ctypes.create_string_buffer(4096)  # (never reached by a launch: every call fails)
    launches = kernels.num_kernel_launches()
    for shift in (11, 19):
        assert lib.elb_cdc_cut(descs, 1, shift, 64, buf, buf, None) == -1
        assert _native.last_error() == "elb_cdc_cut: mean chunk shift %d is not in [12, 18]" % shift
        assert lib.elb_cdc_hash_insert(descs, 1, shift, 64, buf, buf, None, buf, buf, 1024, buf,
                                       None) == -1
        assert _native.last_error() == ("elb_cdc_hash_insert: mean chunk shift %d is not in "
                                        "[12, 18]" % shift)
    assert lib.elb_cdc_cut(descs, 1, 12, 64, None, buf, None) == -1
    assert _native.last_error() == "elb_cdc_cut: NULL descriptor, count or end array"
    assert lib.elb_cdc_cut(None, 1, 12, 64, buf, buf, None) == -1
    assert _native.last_error() == "elb_cdc_cut: NULL descriptor, count or end array"
    # 64K at MIN 1K: up to 64 chunks
    assert lib.elb_cdc_cut(descs, 1, 12, 63, buf, buf, None) == -1
    assert _native.last_error() == ("elb_cdc_cut: descriptor 0 can have 64 chunks, more than 63 "
                                    "slots per descriptor")
    assert lib.elb_cdc_hash_insert(descs, 1, 12, 64, buf, buf, None, buf, buf, 1000, buf,
                                   None) == -1
    assert _native.last_error() == "elb_cdc_hash_insert: table size 1000 is not a power of two"
    assert lib.elb_cdc_hash_insert(descs, 1, 12, 64, buf, buf, None, None, buf, 1024, buf,
                                   None) == -1
    assert _native.last_error() == "elb_cdc_hash_insert: NULL table or counters"
    assert lib.elb_cdc_hash_insert(descs, 1, 12, 64, buf, buf, None, buf, buf, 1024, None,
                                   None) == -1
    assert _native.last_error() == "elb_cdc_hash_insert: NULL table or counters"
    assert lib.elb_cdc_hash_insert(descs, 1, 12, 64, buf, None, None, buf, buf, 1024, buf,
                                   None) == -1
    assert _native.last_error() == ("elb_cdc_hash_insert: NULL payloads, descriptor, count or end "
                                    "array")
    assert lib.elb_cdc_hash_insert(descs, 1, 12, 64, buf, buf, None, buf, None, 1024, buf,
                                   None) == -1
    assert _native.last_error() == ("elb_cdc_hash_insert: NULL payloads, descriptor, count or end "
                                    "array")
    assert lib.elb_cdc_hash_insert(descs, 1, 14, 15, buf, buf, None, buf, buf, 1024, buf,
                                   None) == -1
    assert _native.last_error() == ("elb_cdc_hash_insert: descriptor 0 can have 16 chunks, more "
                                    "than 15 slots per descriptor")
    # nothing to cut or hash: no launch
    assert lib.elb_cdc_cut(None, 0, 12, 64, None, None, None) == 0
    assert lib.elb_cdc_hash_insert(None, 0, 12, 64, None, None, None, buf, buf, 1024, buf,
                                   None) == 0
    assert kernels.num_kernel_launches() == launches


@pytest.mark.parametrize("avg,counts,line", [
    (16 * KiB, (0, 0, 0, 0), "CDC: 0 chunks of 4096 to 65536 bytes, mean 0, 0 distinct: 0 bytes, "
                             "0 distinct bytes: 1.00:1"),
    (16 * KiB, (453, 235, 8388611, 4285825),
     "CDC: 453 chunks of 4096 to 65536 bytes, mean 18517, 235 distinct: 8388611 bytes, 4285825 "
     "distinct bytes: 1.96:1"),
    (4 * KiB, (64, 1, MiB, 16 * KiB), "CDC: 64 chunks of 1024 to 16384 bytes, mean 16384, "
                                       "1 distinct: 1048576 bytes, 16384 distinct bytes: 64.00:1"),
])
def test_console_line(avg, counts, line):
    n, d, b, u = counts
    assert kernels.cdc_line(avg, n, d, b, u) == line == model.line(avg, n, d, b, u)


def test_console_line_needs_counters():
    lib = _native.load()
    assert lib.elb_format_cdc_line(16 * KiB, None, None, 0) == -1
    assert _native.last_error() == "elb_format_cdc_line: NULL counters"
