"""CPU tests of --dedupestats: the command line's rejections, acceptances and help text, the
config's rejections, elb_cfg::dedupeChunkShift at offset 4 of a struct that stays 360 bytes, the
zero-chunk digest against the numpy BLAKE3 model and the `blake3` package, and the argument checks
of elb_dedupe_insert and elb_dedupe_merge."""
import ctypes

import pytest

from elbencho_b200 import WorkerConfig, WorkerError, WorkerManager, _native, kernels
from elbencho_b200.worker import PathType
from tests import blake3_model as model
from tests.test_cli import run_cli

KiB, MiB = 1 << 10, 1 << 20

CLI = ["-w", "-r", "-b", "256k", "-s", "4m", "--gpuids", "0"]


def test_cfg_field_takes_the_hole_at_offset_4():
    assert _native.Cfg.dedupeChunkShift.offset == 4
    assert _native.Cfg.paths.offset == 8
    assert ctypes.sizeof(_native.Cfg) == 360
    assert _native.load().elb_cfg_struct_size() == 360


@pytest.mark.parametrize("size", ["4k", "64k", "256k"])
def test_cli_accepts(tmp_path, size):
    res = run_cli("--dryrun", *CLI, "--dedupestats", size, str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr


@pytest.mark.parametrize("extra,message", [
    (["--dedupestats", "3k"], 'Option "--dedupestats" must be a power of two from 4K to 1G'),
    (["--dedupestats", "2k"], 'Option "--dedupestats" must be a power of two from 4K to 1G'),
    (["--dedupestats", "2g"], 'Option "--dedupestats" must be a power of two from 4K to 1G'),
    (["--dedupestats", "512k"], 'The block size (262144) must be a multiple of "--dedupestats" '
                                '(524288)'),
    (["--dedupestats", "64k", "--rand", "--norandalign"],
     'Option "--dedupestats" cannot be used together with "--norandalign"'),
    (["--dedupestats", "64k", "--rand"],
     'Option "--dedupestats" cannot be used together with "--rand"'),
    (["--dedupestats", "64k", "--infloop"],
     'Option "--dedupestats" cannot be used together with "--infloop"'),
    (["--dedupestats", "64k", "--rwmixpct", "50"],
     'Option "--dedupestats" cannot be used together with "--rwmixpct"'),
    (["--dedupestats", "64k", "--rwmixthr", "1"],
     'Option "--dedupestats" cannot be used together with "--rwmixthr"'),
    (["--dedupestats", "64k", "--hosts", "localhost"],
     'Option "--dedupestats" cannot be used together with "--hosts"'),
])
def test_cli_rejections(tmp_path, extra, message):
    res = run_cli(*CLI, *extra, str(tmp_path / "data"))
    assert res.returncode == 1
    assert message in res.stderr, res.stderr


def test_help_text():
    text = " ".join(run_cli("--help-all").stdout.split())
    assert "--dedupestats arg" in text
    assert ('prints "Dedupe: <N> chunks of <K>, <D> distinct, <Z> zero: <N/D>:1". A file\'s short '
            "last chunk counts as a chunk of its own length. Cannot be used with --rand, "
            "--norandalign, --infloop, --rwmixpct, --rwmixthr or --hosts. [b200]") in text


@pytest.mark.parametrize("extra,message", [
    (dict(dedupe_chunk=2 * KiB), "The dedupe chunk shift (11) is not in [12, 30]."),
    (dict(dedupe_chunk=3 * KiB), "The dedupe chunk shift (-1) is not in [12, 30]."),
    (dict(dedupe_chunk=512 * KiB), "The block size (262144) is not a multiple of the dedupe chunk "
                                   "size (--dedupestats) (524288)."),
    (dict(dedupe_chunk=64 * KiB, use_random_offsets=True),
     "Dedupe stats (--dedupestats) cannot be used together with random offsets: they need every "
     "chunk of a file exactly once."),
    (dict(dedupe_chunk=64 * KiB, do_infinite_io_loop=True),
     "Dedupe stats (--dedupestats) cannot be used together with an infinite I/O loop "
     "(--infloop)."),
    (dict(dedupe_chunk=64 * KiB, rwmix_read_percent=50),
     "Dedupe stats (--dedupestats) cannot be used together with rwmix (a phase in both "
     "directions)."),
    (dict(dedupe_chunk=64 * KiB, num_threads=2, num_rwmix_read_threads=1),
     "Dedupe stats (--dedupestats) cannot be used together with rwmix (a phase in both "
     "directions)."),
])
def test_config_rejections(tmp_path, extra, message):
    cfg = WorkerConfig(paths=[str(tmp_path / "f")], block_size=256 * KiB, file_size=4 * MiB,
                       **extra)
    with pytest.raises(WorkerError) as excinfo:
        WorkerManager(cfg)
    assert str(excinfo.value) == message


def test_config_rejects_norandalign_before_the_random_offsets(tmp_path):
    cfg = WorkerConfig(paths=[str(tmp_path / "f")], block_size=256 * KiB, file_size=4 * MiB,
                       dedupe_chunk=64 * KiB, use_random_unaligned=True)
    with pytest.raises(WorkerError) as excinfo:
        WorkerManager(cfg)
    assert str(excinfo.value) == ("Dedupe stats (--dedupestats) cannot be used together with "
                                  "unaligned random offsets (--norandalign).")


@pytest.mark.parametrize("chunk", [4 * KiB, 64 * KiB, MiB])
def test_zero_digest_matches_model_and_package(chunk):
    got = kernels.dedupe_zero_digest(chunk.bit_length() - 1)
    assert got == model.digest(bytes(chunk))
    blake3 = pytest.importorskip("blake3")
    assert got == blake3.blake3(bytes(chunk)).digest()


@pytest.mark.parametrize("shift", [0, 11, 31, 64])
def test_zero_digest_rejects_shifts(shift):
    with pytest.raises(kernels.KernelError, match=r"chunk shift %d is not in \[12, 30\]" % shift):
        kernels.dedupe_zero_digest(shift)


def test_insert_and_merge_argument_checks():
    lib = _native.load()
    raw = kernels.pack_block_descs([(0x1000, 64 * KiB, 0, 0)])
    descs = ctypes.create_string_buffer(raw, len(raw))
    buf = ctypes.create_string_buffer(4096)  # (never reached by a launch: every call fails)
    zero = kernels.dedupe_zero_digest(12)

    def insert(*args):
        return lib.elb_dedupe_insert(*args)

    assert insert(descs, 1, 12, 16, buf, buf, 1000, buf, zero, None) == -1
    assert _native.last_error() == "elb_dedupe_insert: table size 1000 is not a power of two"
    assert insert(descs, 1, 12, 16, buf, buf, 0, buf, zero, None) == -1
    assert _native.last_error() == "elb_dedupe_insert: table size 0 is not a power of two"
    assert insert(descs, 1, 12, 16, buf, None, 1024, buf, zero, None) == -1
    assert _native.last_error() == "elb_dedupe_insert: NULL table or counters"
    assert insert(descs, 1, 12, 16, buf, buf, 1024, None, zero, None) == -1
    assert _native.last_error() == "elb_dedupe_insert: NULL table or counters"
    for args in [(None, 1, 12, 16, buf), (descs, 1, 12, 16, None)]:
        assert insert(*args, buf, 1024, buf, zero, None) == -1
        assert _native.last_error() == ("elb_dedupe_insert: NULL descriptor, digest or zero "
                                        "digest array")
    assert insert(descs, 1, 12, 16, buf, buf, 1024, buf, None, None) == -1
    for shift in (11, 31, 64):
        assert insert(descs, 1, shift, 16, buf, buf, 1024, buf, zero, None) == -1
        assert _native.last_error() == ("elb_dedupe_insert: chunk shift %d is not in [12, 30]"
                                        % shift)
    off = kernels.pack_block_descs([(0x1000, 64 * KiB, 2 * KiB, 0)])
    off_descs = ctypes.create_string_buffer(off, len(off))
    assert insert(off_descs, 1, 12, 16, buf, buf, 1024, buf, zero, None) == -1
    assert _native.last_error() == ("elb_dedupe_insert: descriptor 0 (offset 2048) is not on a "
                                    "chunk boundary")
    assert insert(descs, 1, 12, 15, buf, buf, 1024, buf, zero, None) == -1
    assert _native.last_error() == ("elb_dedupe_insert: descriptor 0 has 16 chunks, more than 15 "
                                    "slots per descriptor")
    # nothing to insert: no launch
    assert insert(None, 0, 12, 16, None, buf, 1024, buf, zero, None) == 0

    assert lib.elb_dedupe_merge(buf, 16, buf, 3, buf, None) == -1
    assert _native.last_error() == "elb_dedupe_merge: table size 3 is not a power of two"
    assert lib.elb_dedupe_merge(buf, 16, None, 1024, buf, None) == -1
    assert _native.last_error() == "elb_dedupe_merge: NULL table or counters"
    assert lib.elb_dedupe_merge(None, 16, buf, 1024, buf, None) == -1
    assert _native.last_error() == "elb_dedupe_merge: NULL source entries"
    assert lib.elb_dedupe_merge(None, 0, buf, 1024, buf, None) == 0


def test_stats_need_the_option():
    lib = _native.load()
    out = [ctypes.c_uint64(7) for _ in range(3)]
    assert lib.elb_mgr_dedupe_stats(None, *[ctypes.byref(v) for v in out]) == -1
    assert _native.last_error() == "elb_mgr_dedupe_stats: NULL argument"


@pytest.mark.parametrize("mode", ["file", "dir"])
def test_dry_run_with_other_options(tmp_path, mode):
    extra = ["-d", "-n", "2", "-N", "3"] if mode == "dir" else []
    res = run_cli("--dryrun", *CLI, *extra, "--dedupestats", "64k", "--checksums",
                  str(tmp_path / "sums"), "--checksumalgo", "blake3", "--checksumchunk", "64k",
                  str(tmp_path if mode == "dir" else tmp_path / "data"))
    assert res.returncode == 0, res.stderr


def test_dir_mode_config_is_accepted(tmp_path):
    # (the table is made at the start of a phase: creating the manager allocates nothing for it)
    cfg = WorkerConfig(paths=[str(tmp_path)], path_type=PathType.DIR, num_dirs=1, num_files=1,
                       block_size=64 * KiB, file_size=64 * KiB, dedupe_chunk=4 * KiB)
    assert cfg.to_abi()[0].dedupeChunkShift == 12


@pytest.mark.parametrize("block,size", [("96k", "64k"), ("1m", "100k")])
def test_block_reduced_to_the_file_size_is_accepted(tmp_path, block, size):
    """a block larger than the file is the whole file (its last chunk may be short), for the
    command line as for the config"""
    res = run_cli("--dryrun", "-w", "-b", block, "-s", size, "--gpuids", "0", "--dedupestats",
                  "64k", str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr
    res = run_cli("--dryrun", "-w", "-b", "96k", "-s", "1m", "--gpuids", "0", "--dedupestats",
                  "64k", str(tmp_path / "data"))
    assert res.returncode == 1
    assert 'The block size (98304) must be a multiple of "--dedupestats" (65536)' in res.stderr
