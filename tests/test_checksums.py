"""CPU tests of --checksums: the CRC model against zlib, the library's shift and finish against
the model, the command line and config rejections, the help text, a dry run and the elb_cfg
field."""
import ctypes
import random
import zlib

import pytest

from elbencho_b200 import WorkerConfig, WorkerError, WorkerManager, _native, kernels
from tests import crc_model as model
from tests.test_cli import run_cli

MiB = 1 << 20

CLI = ["-w", "-r", "-b", "1m", "-s", "16m", "--gpuids", "0"]


@pytest.mark.parametrize("seed", range(40))
def test_model_matches_zlib_for_random_splits(seed):
    rng = random.Random(seed)
    size = rng.choice([0, 1, 2, 15, 16, 17, 255, 4096, rng.randint(0, 20000)])
    data = rng.randbytes(size)
    parts = model.random_split(size, rng)

    assert sum(length for _, length in parts) == size
    assert model.finish(model.file_raw_crc(data, parts), size) == zlib.crc32(data)


def test_model_shift_appends_zero_bytes():
    rng = random.Random(7)
    for n in (0, 1, 3, 64, 1000):
        data = rng.randbytes(rng.randint(1, 50))
        assert model.shift(model.raw_crc(data), n) == model.raw_crc(data + bytes(n))


@pytest.mark.parametrize("n", [0, 1, 2, 7, 8, 4095, 4096, 1 << 20, (1 << 32) - 2, (1 << 32) - 1,
                               1 << 32, (1 << 32) + 5, 5 << 30, (1 << 63) + 12345,
                               (1 << 64) - 1])
def test_library_shift_matches_model(n):
    for crc in (0, 1, 0x80000000, 0xFFFFFFFF, 0x12345678):
        assert kernels.crc32_shift(crc, n) == model.shift(crc, n)


@pytest.mark.parametrize("size", [0, 1, 5, 4096, (1 << 32) + 3, 1 << 40])
def test_library_finish_matches_model(size):
    for raw in (0, 0xDEADBEEF):
        assert kernels.crc32_finish(raw, size) == model.finish(raw, size)


def test_library_finish_is_zlib():
    data = random.Random(3).randbytes(3000)
    assert kernels.crc32_finish(model.raw_crc(data), len(data)) == zlib.crc32(data)


@pytest.mark.parametrize("extra,message", [
    (["--rand"], 'Option "--checksums" cannot be used together with "--rand"'),
    (["--infloop", "--timelimit", "1"],
     'Option "--checksums" cannot be used together with "--infloop"'),
    (["--rwmixpct", "20"], 'Option "--checksums" cannot be used together with "--rwmixpct"'),
    (["--rwmixthr", "1", "-t", "2"],
     'Option "--checksums" cannot be used together with "--rwmixthr"'),
    (["--hosts", "localhost:1"], 'Option "--checksums" cannot be used together with "--hosts"'),
])
def test_validation_messages(extra, message):
    res = run_cli(*CLI, *extra, "--checksums", "/tmp/elb_checksums", "/tmp/x")
    assert res.returncode == 1
    assert message in res.stderr, res.stderr


@pytest.mark.parametrize("args", [
    [], ["--verify", "3"], ["--verifyrand", "3", "--verifyrandgrain", "64k"],
    ["--blockvarpct", "100"], ["--verify", "3", "--verifydirect"],
])
def test_accepted_combinations(args, tmp_path):
    res = run_cli("--dryrun", *CLI, *args, "--checksums", str(tmp_path / "sums"),
                  str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr


def test_help_lists_the_option():
    res = run_cli("--help-all")
    assert res.returncode == 0
    text = " ".join(res.stdout.split())
    assert "--checksums" in text
    assert "# phase WRITE|READ" in text
    assert "Cannot be used with --rand, --infloop, --rwmixpct, --rwmixthr or --hosts." in text


def test_cfg_field_fills_padding():
    assert ctypes.sizeof(_native.Cfg) == _native.load().elb_cfg_struct_size() == 360
    assert _native.Cfg.ioEngine.offset == 64
    assert _native.Cfg.checksumReport.offset == 68
    assert _native.Cfg.numDirs.offset == 72


@pytest.mark.parametrize("kwargs,message", [
    (dict(use_random_offsets=True),
     "Checksums (--checksums) cannot be used together with random offsets: they need every "
     "block of a file exactly once."),
    (dict(do_infinite_io_loop=True),
     "Checksums (--checksums) cannot be used together with an infinite I/O loop (--infloop)."),
    (dict(rwmix_read_percent=10),
     "Checksums (--checksums) cannot be used together with rwmix (a phase in both directions)."),
])
def test_config_rejection(tmp_path, kwargs, message):
    cfg = WorkerConfig(paths=[str(tmp_path / "f")], block_size=MiB, file_size=MiB,
                       checksums=True, **kwargs)
    with pytest.raises(WorkerError) as excinfo:
        WorkerManager(cfg)
    assert str(excinfo.value) == message


def test_crc32_blocks_argument_checks():
    lib = _native.load()
    assert lib.elb_crc32_blocks(None, None, 1, None, None, None, None) == -1
    assert "NULL descriptor, shift or CRC array" in _native.last_error()

    raw = kernels.pack_block_descs([(0x1000, 16, 0, 0)])
    descs = ctypes.create_string_buffer(raw, len(raw))
    shifts = (ctypes.c_uint64 * 1)(0)
    crcs = (ctypes.c_uint32 * 1)(0)
    assert lib.elb_crc32_blocks(descs, shifts, 1, crcs, crcs, None, None) == -1
    assert "host CRCs and device ticket go together" in _native.last_error()

    assert lib.elb_crc32_blocks(None, None, 0, None, None, None, None) == 0
