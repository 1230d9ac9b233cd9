"""CPU tests of --verifyreport: the command line and config rejections, the elb_cfg field, the
argument checks of elb_damage_map (exact texts, in order, no launch), and the merge rule of the
model (tests/verify_report_model.py) on handmade cases."""
import ctypes

import pytest

from elbencho_b200 import WorkerConfig, WorkerError, WorkerManager, _native, kernels
from tests import verify_report_model as model
from tests.test_cli import run_cli

KiB, MiB = 1 << 10, 1 << 20

CLI = ["-r", "-b", "1m", "-s", "16m", "--gpuids", "0"]


@pytest.mark.parametrize("args,message", [
    (CLI + ["--verifyreport", "/tmp/elb_report", "/tmp/x"],
     'Option "--verifyreport" requires "--verify" or "--verifyrand"'),
    (CLI + ["--verify", "3", "--verifyreport", "/tmp/elb_report", "--hosts", "localhost:1",
            "/tmp/x"],
     'Option "--verifyreport" cannot be used together with "--hosts"'),
    (CLI + ["--verifyrand", "3", "--verifyreport", "/tmp/elb_report", "--hosts", "a:1,b:2",
            "/tmp/x"],
     'Option "--verifyreport" cannot be used together with "--hosts"'),
])
def test_validation_messages(args, message):
    res = run_cli(*args)
    assert res.returncode == 1
    assert message in res.stderr, res.stderr


@pytest.mark.parametrize("args", [
    ["--verify", "3"], ["--verifyrand", "3"], ["--verifyrand", "3", "--verifyrandgrain", "64k"],
    ["--verifyrand", "3", "--verifyrandgrain", "64k", "--dedupepct", "20"],
])
def test_accepted_combinations(args):
    res = run_cli("--dryrun", *CLI, *args, "--verifyreport", "/tmp/elb_dry_report",
                  "/tmp/elb_dry_report_file")
    assert res.returncode == 0, res.stderr


def test_help_lists_the_option():
    res = run_cli("--help-all")
    assert res.returncode == 0
    assert "--verifyreport" in " ".join(res.stdout.split())


def test_cfg_field_fills_padding():
    assert ctypes.sizeof(_native.Cfg) == _native.load().elb_cfg_struct_size() == 360
    assert _native.Cfg.randOffsetAlgo.offset == 232
    assert _native.Cfg.verifyDamageReport.offset == 236
    assert _native.Cfg.limitReadBps.offset == 240


def test_config_rejection(tmp_path):
    cfg = WorkerConfig(paths=[str(tmp_path / "f")], block_size=MiB, file_size=MiB,
                       verify_report=True)
    with pytest.raises(WorkerError) as excinfo:
        WorkerManager(cfg)
    assert str(excinfo.value) == ("A verify report (--verifyreport) requires data verification "
                                  "(--verify or --verifyrand).")


# ---- elb_damage_map argument checks ------------------------------------------------------------

def descs(*blocks):
    """pinned-host stand-in: ordinary host memory is enough for checks that end before a launch"""
    raw = kernels.pack_block_descs(blocks)
    return ctypes.create_string_buffer(raw, len(raw))


@pytest.mark.parametrize("args,message", [
    # (kind, key, pct, grainShift, dedupePct, sectors, sectorsPerDesc)
    ((0, 1, 0, 0, 0), "elb_damage_map: unknown content kind: 0"),
    ((4, 1, 0, 0, 0), "elb_damage_map: unknown content kind: 4"),
    ((kernels.CONTENT_RANDOM_GRAIN, 1, 101, 11, 101),
     "Random verify grain shift must be in range 12..30. Given: 11"),
    ((kernels.CONTENT_RANDOM_GRAIN, 1, 101, 31, 0),
     "Random verify grain shift must be in range 12..30. Given: 31"),
    ((kernels.CONTENT_RANDOM_GRAIN, 1, 101, 12, 101),
     "Block variance percent must be in range 0..100. Given: 101"),
    ((kernels.CONTENT_RANDOM, 1, 101, 0, 0),
     "Block variance percent must be in range 0..100. Given: 101"),
    ((kernels.CONTENT_RANDOM_GRAIN, 1, 100, 12, 101),
     "Dedupe percent must be in range 0..100. Given: 101"),
    ((kernels.CONTENT_PATTERN, 1, 0, 0, 200), "Dedupe percent must be in range 0..100. Given: 200"),
])
def test_content_checks_in_order(native, args, message):
    before = native.elb_num_kernel_launches()
    buf = descs((0x1000, 4096, 0, 0))
    res = native.elb_damage_map(buf, 1, *args, 0x2000, 8, None)
    assert res == -1
    assert _native.last_error() == message
    assert native.elb_num_kernel_launches() == before


def test_pointer_and_size_checks(native):
    before = native.elb_num_kernel_launches()
    pattern = (kernels.CONTENT_PATTERN, 1, 0, 0, 0)
    assert native.elb_damage_map(None, 1, *pattern, 0x2000, 8, None) == -1
    assert _native.last_error() == "elb_damage_map: NULL descriptor or sector array"
    assert native.elb_damage_map(descs((0x1000, 4096, 0, 0)), 1, *pattern, None, 8, None) == -1
    assert _native.last_error() == "elb_damage_map: NULL descriptor or sector array"
    # a 4 KiB block at offset 100 touches 9 sectors; the second descriptor is rejected by index
    buf = descs((0x1000, 4096, 0, 0), (0x3000, 4096, 100, 0))
    assert native.elb_damage_map(buf, 2, *pattern, 0x9000, 8, None) == -1
    assert _native.last_error() == ("elb_damage_map: descriptor 1 touches 9 sectors, more than "
                                    "sectorsPerDesc (8)")
    # one byte before a sector boundary plus one after: 2 sectors
    assert native.elb_damage_map(descs((0x1000, 2, 511, 0)), 1, *pattern, 0x9000, 1,
                                 None) == -1
    assert _native.last_error() == ("elb_damage_map: descriptor 0 touches 2 sectors, more than "
                                    "sectorsPerDesc (1)")
    # nothing to do: no descriptors, or only empty ones
    assert native.elb_damage_map(None, 0, *pattern, None, 0, None) == 0
    assert native.elb_damage_map(descs((0x1000, 0, 7, 0)), 1, *pattern, 0x9000, 0, None) == 0
    assert native.elb_num_kernel_launches() == before


# ---- the model's merge rule on handmade cases --------------------------------------------------

def damaged(size, positions, value=0):
    expected = bytes(size)
    actual = bytearray(expected)
    for pos in positions:
        actual[pos] = value ^ 0x5A
    return expected, bytes(actual)


def test_single_byte_and_sector_boundary_run():
    files = {"f": damaged(8 * KiB, [700, 1020, 1021, 1022, 1023, 1024, 1025, 3000])}
    lines = model.extents(files, {"f": [(0, 8 * KiB)]})
    # 700 (sector 1), 1020..1025 (sectors 1, 2): one extent; 3000 (sector 5) another
    assert lines == [("f", 700, 1025 - 700 + 1, 7), ("f", 3000, 1, 1)]


def test_sector_read_twice_counts_once():
    files = {"f": damaged(4 * KiB, [10, 11, 600])}
    once = model.extents(files, {"f": [(0, 4 * KiB)]})
    twice = model.extents(files, {"f": [(0, 4 * KiB), (0, 4 * KiB), (0, 1 * KiB)]})
    assert once == twice == [("f", 10, 591, 3)]


def test_sector_split_between_blocks_adds_up():
    """-b 1000: sector 1 (bytes 512..1023) is read in two parts by two blocks"""
    files = {"f": damaged(3000, [900, 999, 1000, 1010])}
    lines = model.extents(files, {"f": [(0, 1000), (1000, 1000), (2000, 1000)]})
    assert lines == [("f", 900, 111, 4)]
    # and a re-read of one part still counts once
    again = model.extents(files, {"f": [(0, 1000), (1000, 1000), (2000, 1000), (1000, 1000)]})
    assert again == lines


def test_runs_merge_across_blocks_and_workers():
    """damage in the last sector of one block and the first of the next, read by two workers in
    either order: one extent; a clean sector in between splits it"""
    files = {"a": damaged(8 * KiB, [4095, 4096, 4097]),
             "b": damaged(8 * KiB, [4095, 4608])}
    ranges = {"a": [(4096, 4096), (0, 4096)], "b": [(0, 4096), (4096, 4096)]}
    assert model.extents(files, ranges) == [("a", 4095, 3, 3), ("b", 4095, 1, 1),
                                            ("b", 4608, 1, 1)]


def test_unread_bytes_do_not_count():
    files = {"f": damaged(4 * KiB, [100, 2000])}
    assert model.extents(files, {"f": [(1024, 1024)]}) == [("f", 2000, 1, 1)]
    assert model.extents(files, {"f": []}) == []


def test_truncation_counts_runs_before_the_merge():
    """a worker lists its first runs only (here 2), counted per block before the merge"""
    exp, act = damaged(16 * KiB, [0, 1024, 5000, 9000, 9001])
    blocks = [model.sector_records(exp, act, [(off, 4 * KiB)]) for off in range(0, 16 * KiB,
                                                                                 4 * KiB)]
    listed, dropped_runs, dropped_bytes = model.truncate_runs(blocks, 2)
    assert (dropped_runs, dropped_bytes) == (2, 3)
    lines = model.merge({"f": listed})
    assert lines == [("f", 0, 1, 1), ("f", 1024, 1, 1)]
    assert model.report_text(lines, dropped_runs, dropped_bytes) == (
        "f\t0\t1\t1\nf\t1024\t1\t1\n# truncated: 2 more extents, 3 differing bytes not listed\n")


def test_pattern_content_closed_form():
    raw = model.pattern_content(0, 24, 5)
    assert raw[:8] == (5).to_bytes(8, "little") and raw[8:16] == (13).to_bytes(8, "little")
    assert model.pattern_content(3, 10, 5) == raw[3:13]
