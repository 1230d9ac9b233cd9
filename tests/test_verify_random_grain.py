"""CPU tests of --verifyrandgrain: the grain model against the per-block --verifyrand content it
extends, known-answer bytes at the grain, part and 2^64 edges, the command line option and the
config with their rejections, the service key, and the elb_cfg field that carries the grain."""
import ctypes

import numpy as np
import pytest

from elbencho_b200 import WorkerConfig, WorkerError, WorkerManager, _native, kernels
from tests import verify_random_grain_model as model
from tests import verify_random_model as vrm
from tests.test_cli import run_cli
from tests.test_master_fake_services import FakeService, run_master

KiB, MiB = 1 << 10, 1 << 20
U64 = model.U64


@pytest.mark.parametrize("grain,pct", [(4 * KiB, 100), (32 * KiB, 33), (64 * KiB, 50),
                                       (4 * KiB, 0)])
def test_model_equals_per_block_content_at_block_size_grain(grain, pct):
    """a file written per block with -b G in full blocks is the grain-mode file of G"""
    for key in (0, 3, vrm.dir_file_key(1, 2, 3)):
        size = 5 * grain
        assert model.file_content(size, grain, pct, 0xBEEF, key) == \
            vrm.file_random_content(size, grain, pct, 0xBEEF, key)


# (position, grain, pct, seed, fileKey) -> byte
GRAIN_BYTE_KAT = [
    ((4095, 4096, 100, 7, 0), 61),             # last byte of grain 0
    ((4096, 4096, 100, 7, 0), 168),            # first byte of grain 1
    ((0, 1 << 15, 33, 0xABC, 5), 238),
    ((10811, 1 << 15, 33, 0xABC, 5), 5),       # last random byte (varFill 10812, = 4 mod 8)
    ((10812, 1 << 15, 33, 0xABC, 5), 178),     # first remainder byte
    ((U64, 4096, 50, 99, 3), 14),              # the last byte before 2^64 ...
    ((0, 4096, 50, 99, 3), 226),               # ... and the first after it
]


@pytest.mark.parametrize("args,want", GRAIN_BYTE_KAT)
def test_known_answer_bytes(args, want):
    pos, grain, pct, seed, key = args
    assert model.content(pos, 1, grain, pct, seed, key)[0] == want


def test_content_across_the_wrap():
    """8 bytes from 2^64 - 4 are the last 4 of the top grain and the first 4 of grain 0"""
    assert model.content(U64 - 3, 8, 4096, 100, 1, 2).hex() == "2901932ef677cc86"
    top = model.grain_bytes(4096, 100, 1, 2, (U64 + 1) - 4096)
    assert model.content(U64 - 3, 8, 4096, 100, 1, 2) == \
        top[-4:] + model.grain_bytes(4096, 100, 1, 2, 0)[:4]


def test_random_and_remainder_parts_of_a_grain():
    grain, pct = 32 * KiB, 33
    var = grain * pct // 100 // 4 * 4
    data = np.frombuffer(model.grain_bytes(grain, pct, 5, 6, 3 * grain), dtype=np.uint8)
    rem = np.frombuffer(data[var:var + 8].tobytes(), dtype=np.uint64)[0]
    # the remainder is one repeated u64, starting at varFill
    assert np.all(np.frombuffer(data[var:var + (grain - var) // 8 * 8].tobytes(),
                                dtype=np.uint64) == rem)


def test_error_text_model():
    grain, pct, seed = 4 * KiB, 100, 99
    data = bytearray(model.file_content(3 * grain + 100, grain, pct, seed, 0))
    assert model.error_text(bytes(data), grain, pct, seed, 0) is None
    data[5000] ^= 1
    want = model.content(5000, 1, grain, pct, seed, 0)[0]
    assert model.error_text(bytes(data), grain, pct, seed, 0) == (
        "Data verification failed. Offset: 5000; Expected value: %d; Actual value: %d"
        % (want, want ^ 1))


# ---- C ABI -------------------------------------------------------------------------------------

def test_cfg_field_replaces_a_reserved_int():
    lib = _native.load()
    assert lib.elb_cfg_struct_size() == ctypes.sizeof(_native.Cfg) == 360
    assert lib.elb_abi_version() == 1
    assert _native.Cfg._fields_[-1][0] == "integrityCheckKind"
    assert _native.Cfg.randomVerifyGrainShift.offset == 292
    assert "reserved4" not in [f[0] for f in _native.Cfg._fields_]


def base_cfg(tmp_path, **kwargs):
    cfg = dict(paths=[str(tmp_path / "f")], block_size=4096, file_size=MiB,
               integrity_check_salt=5, integrity_check_kind=kernels.VERIFY_RANDOM,
               block_variance_percent=100, verify_random_grain=64 * KiB)
    cfg.update(kwargs)
    return WorkerConfig(**cfg)


@pytest.mark.parametrize("kwargs,message", [
    (dict(verify_random_grain=2 * KiB), "Invalid random verify grain shift: 11 (0 or 12..30)"),
    (dict(verify_random_grain=2 << 30), "Invalid random verify grain shift: 31 (0 or 12..30)"),
    (dict(verify_random_grain=5000), "Invalid random verify grain shift: -1 (0 or 12..30)"),
    (dict(integrity_check_kind=kernels.VERIFY_PATTERN),
     "A random verify grain (--verifyrandgrain) requires random data verification "
     "(--verifyrand)."),
    (dict(integrity_check_salt=0),
     "A random verify grain (--verifyrandgrain) requires random data verification "
     "(--verifyrand)."),
    (dict(rwmix_read_percent=10), "Integrity check cannot be used together with rwmixpct."),
])
def test_config_rejections(tmp_path, kwargs, message):
    with pytest.raises(WorkerError) as excinfo:
        WorkerManager(base_cfg(tmp_path, **kwargs))
    assert str(excinfo.value) == message


def test_config_rejects_unaligned_random_offsets_per_block_only(tmp_path):
    """(the worker tests on the GPU read grain-mode files at unaligned random offsets)"""
    unaligned = dict(use_random_offsets=True, use_random_unaligned=True, rand_offset_seed=1)
    with pytest.raises(WorkerError) as excinfo:
        WorkerManager(base_cfg(tmp_path, verify_random_grain=0, **unaligned))
    assert str(excinfo.value) == ("Random data verification (--verifyrand) cannot be used "
                                  "together with unaligned random offsets.")


# ---- command line ------------------------------------------------------------------------------

def test_help_describes_the_option():
    res = run_cli("--help")
    assert res.returncode == 0
    text = " ".join(res.stdout.split())
    assert "--verifyrandgrain" in text
    assert "reads of any block size and offset" in text
    assert "Writes and reads must use the same value" in text
    assert "not block size independent" in text  # (--verifyrand's own text stays)


GRAIN_RANGE = 'Option "--verifyrandgrain" must be a power of two from 4K to 1G'


@pytest.mark.parametrize("args,message", [
    (["-w", "-s", "1g", "--gpuids", "0", "--verifyrandgrain", "64k", "/tmp/x"],
     'Option "--verifyrandgrain" requires "--verifyrand"'),
    (["-w", "-s", "1g", "--gpuids", "0", "--verify", "3", "--verifyrandgrain", "64k", "/tmp/x"],
     'Option "--verifyrandgrain" requires "--verifyrand"'),
    (["-w", "-s", "1g", "--gpuids", "0", "--verifyrand", "2", "--verifyrandgrain", "48k",
      "/tmp/x"], GRAIN_RANGE),
    (["-w", "-s", "1g", "--gpuids", "0", "--verifyrand", "2", "--verifyrandgrain", "2k",
      "/tmp/x"], GRAIN_RANGE),
    (["-w", "-s", "1g", "--gpuids", "0", "--verifyrand", "2", "--verifyrandgrain", "2g",
      "/tmp/x"], GRAIN_RANGE),
    # the rejections of --verifyrand stay
    (["-w", "-s", "1g", "--gpuids", "0", "--rand", "--verifyrand", "2", "--verifyrandgrain",
      "64k", "/tmp/x"], "Integrity check writes are not supported in combination with random "
     "offsets."),
    (["-w", "-s", "1g", "--gpuids", "0", "--verifyrand", "2", "--verifyrandgrain", "64k",
      "--rwmixpct", "10", "/tmp/x"],
     'Option --rwmixpct cannot be used together with option "--verifyrand"'),
    (["-w", "-s", "1g", "--gpuids", "0", "--verifyrand", "2", "--verifyrandgrain", "64k",
      "--treefile", "/tmp/t.txt", "/tmp"],
     "Custom tree mode cannot be used together with --verifyrand."),
])
def test_validation_messages(args, message):
    res = run_cli(*args)
    assert res.returncode == 1
    assert message in res.stderr, res.stderr


@pytest.mark.parametrize("args", [
    ["-w", "-r", "-b", "1M", "-s", "16M", "--verifyrand", "7", "--verifyrandgrain", "64K"],
    ["-r", "-b", "4K", "-s", "16M", "--verifyrand", "7", "--verifyrandgrain", "64K", "--rand",
     "--iodepth", "64"],
    ["-r", "-b", "4K", "-s", "16M", "--verifyrand", "7", "--verifyrandgrain", "4K", "--rand",
     "--norandalign"],
    ["-w", "-b", "1000", "-s", "16M", "--verifyrand", "7", "--verifyrandgrain", "1G",
     "--blockvarpct", "50", "--verifydirect"],
])
def test_accepted_combinations(args):
    res = run_cli("--dryrun", *args, "--gpuids", "0", "/tmp/elb_dry_vrg")
    assert res.returncode == 0, res.stderr


def test_grain_travels_to_services(tmp_path):
    svc = FakeService(8 * MiB, [1000, 2000]).start()
    try:
        res = run_master("-w", "-r", "-t", "2", "-b", "1M", "-s", "8M", "--verifyrand", "77",
                         "--verifyrandgrain", "64K", "--gpuids", "0", "--hosts",
                         "127.0.0.1:%d" % svc.port, "--nolive", str(tmp_path / "bench"))
        assert res.returncode == 0, res.stdout + res.stderr
        prep = svc.prepare_trees[0]
        assert prep["b200_verifyrandgrain"] == str(64 * KiB)
        assert prep["b200_verifyrand"] == "77"
    finally:
        svc.stop()
    plain = FakeService(8 * MiB, [1000, 2000]).start()
    try:
        res = run_master("-w", "-t", "2", "-b", "1M", "-s", "8M", "--verifyrand", "77",
                         "--gpuids", "0", "--hosts", "127.0.0.1:%d" % plain.port, "--nolive",
                         str(tmp_path / "bench"))
        assert res.returncode == 0, res.stdout + res.stderr
        assert plain.prepare_trees[0]["b200_verifyrandgrain"] == "0"
    finally:
        plain.stop()
