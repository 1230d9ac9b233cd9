"""CPU tests of --dedupepct: the model (tests/dedupe_model.py) against the library's grain key, the
identity with --verifyrandgrain at 0 percent, the share of duplicate grains and the distinct grain
count against the formula of DESIGN.md, the C ABI's argument checks, the config and command line
rejections, and the service key."""
import random

import numpy as np
import pytest

from elbencho_b200 import WorkerConfig, WorkerError, WorkerManager, _native, kernels
from tests import dedupe_model as model
from tests import kernel_cases as kc
from tests import verify_random_grain_model as vrg
from tests import verify_random_model as vrm
from tests.test_cli import run_cli
from tests.test_master_fake_services import FakeService, run_master

KiB, MiB = 1 << 10, 1 << 20
U64 = model.U64


def key_cases():
    """(seed, fileKey, grainOffset, grainShift, dedupePct): seeded, with the edge values"""
    rng = random.Random(4711)
    for i in range(400):
        shift = rng.choice([12, 13, 16, 20, 29, 30, rng.randrange(12, 31)])
        off = rng.choice([rng.getrandbits(64), U64 + 1 - (rng.randrange(1, 64) << shift),
                          rng.randrange(64) << shift, 0])
        off &= U64 & ~((1 << shift) - 1)
        pct = rng.choice([0, 1, 50, 99, 100, rng.randrange(101)])
        seed = rng.choice([0, 1, U64, rng.getrandbits(64)])
        file_key = rng.choice([0, 3, U64, vrm.dir_file_key(1, 2, 3), rng.getrandbits(64)])
        yield seed, file_key, off, shift, pct


def test_model_key_equals_library_key():
    cases = list(key_cases())
    assert {c[4] for c in cases} >= {0, 100} and {c[3] for c in cases} >= {12, 30}
    assert any(c[2] > U64 - (1 << 36) for c in cases)
    for seed, file_key, off, shift, pct in cases:
        assert kernels.rand_grain_content_key(seed, file_key, off, shift, pct) == \
            model.grain_key(seed, file_key, off, shift, pct), (seed, file_key, off, shift, pct)


def test_zero_percent_is_the_grain_key_of_every_grain():
    for shift in (12, 16, 30):
        for i in range(64):
            off = (i << shift) & U64
            for file_key in (0, 7):
                want = kc.rand_block_key(0xBEEF, vrm.pos_counter(file_key, off))
                assert kernels.rand_grain_content_key(0xBEEF, file_key, off, shift, 0) == want
                assert model.grain_key(0xBEEF, file_key, off, shift, 0) == want
    # (the top grain below 2^64 too)
    top = U64 + 1 - (1 << 12)
    assert kernels.rand_grain_content_key(1, 2, top, 12, 0) == \
        kc.rand_block_key(1, vrm.pos_counter(2, top))


def test_zero_percent_content_is_grain_content():
    for grain, pct in ((4 * KiB, 100), (64 * KiB, 33)):
        assert model.file_content(3 * grain + 5, grain, pct, 0, 9, 4) == \
            vrg.file_content(3 * grain + 5, grain, pct, 9, 4)


def test_hundred_percent_every_grain_is_a_pool_grain():
    grain, pct, seed = 4 * KiB, 50, 0x51
    data = model.file_content(16 * grain, grain, pct, 100, seed, 3)
    for g in range(16):
        s = model.draw(3, g * grain)
        assert model.is_shared(s, 100)
        assert data[g * grain:(g + 1) * grain] == model.pool_grain(grain, pct, seed,
                                                                   model.pool_slot(s))


def draws(num_grains, file_keys=(0,), shift=16):
    """numpy: s of grains 0..num_grains-1 of each file"""
    out = []
    for key in file_keys:
        base = kc._mix(np.uint64((key + vrm.GOLDEN) & U64))
        offs = np.arange(num_grains, dtype=np.uint64) << np.uint64(shift)
        with np.errstate(over="ignore"):
            out.append(kc._mix(kc._mix(base ^ offs) + np.uint64(model.DEDUPE_TAG)))
    return np.concatenate(out)


def test_numpy_draws_equal_the_model():
    s = draws(100, (0, 5))
    assert [int(x) for x in s[:100]] == [model.draw(0, i << 16) for i in range(100)]
    assert int(s[150]) == model.draw(5, 50 << 16)


@pytest.mark.parametrize("pct", [1, 50, 99])
def test_shared_share_is_within_one_point(pct):
    s = draws(10 ** 5)
    shared = ((s >> np.uint64(32)) * np.uint64(100)) >> np.uint64(32) < np.uint64(pct)
    assert abs(100.0 * shared.mean() - pct) < 1.0
    # (the 0..99 draw itself is close to uniform)
    counts = np.bincount(((s >> np.uint64(32)) * np.uint64(100) >> np.uint64(32)).astype(np.int64),
                         minlength=100)
    assert counts.min() > 850 and counts.max() < 1150  # (binomial: sigma 31.5)


@pytest.mark.parametrize("num_grains,pct,files", [(10 ** 4, 1, 1), (10 ** 4, 50, 1),
                                                  (10 ** 5, 50, 1), (10 ** 4, 99, 1),
                                                  (4096, 50, 2), (2000, 30, 4)])
def test_distinct_count_matches_the_formula(num_grains, pct, files):
    per_file = num_grains // files
    grains = [(key, g << 16) for key in range(files) for g in range(per_file)]
    exact = model.distinct_grains(grains, pct)
    assert abs(exact - model.expected_distinct_grains(len(grains), pct)) < 0.01 * exact


def test_distinct_count_edges():
    grains = [(0, g << 12) for g in range(5000)]
    assert model.distinct_grains(grains, 0) == 5000
    assert model.expected_distinct_grains(5000, 0) == 5000
    assert model.distinct_grains(grains, 100) <= model.POOL_GRAINS


def test_error_text_model():
    grain, pct, seed = 4 * KiB, 100, 99
    data = bytearray(model.file_content(3 * grain + 100, grain, pct, 50, seed, 0))
    assert model.error_text(bytes(data), grain, pct, 50, seed, 0) is None
    data[5000] ^= 1
    want = model.content(5000, 1, grain, pct, 50, seed, 0)[0]
    assert model.error_text(bytes(data), grain, pct, 50, seed, 0) == (
        "Data verification failed. Offset: 5000; Expected value: %d; Actual value: %d"
        % (want, want ^ 1))


# ---- C ABI -------------------------------------------------------------------------------------

N, P = None, 0x1000
DEDUPE_FORMS = {
    "elb_fill_dedupe_grain": lambda sh, pct, dp: (N, 0, 0, sh, pct, dp, 1, 2, N),
    "elb_verify_dedupe_grain": lambda sh, pct, dp: (N, 0, 0, sh, pct, dp, 1, 2, P, N),
    "elb_fill_dedupe_grain_batch_sized": lambda sh, pct, dp: (N, 0, sh, pct, dp, 1, N, 0, 0, N),
    "elb_verify_dedupe_grain_batch_sized":
        lambda sh, pct, dp: (N, 0, sh, pct, dp, 1, N, N, 0, 0, N),
    "elb_fill_dedupe_grain_staged": lambda sh, pct, dp: (N, 0, sh, pct, dp, 1, 64, N, 0, 0, N),
    "elb_verify_dedupe_grain_staged":
        lambda sh, pct, dp: (N, 0, sh, pct, dp, 1, 64, N, N, N, N, 0, 0, N),
}


def test_dedupe_table_has_every_entry_point():
    assert sorted(DEDUPE_FORMS) == sorted(n for n in _native.SIGNATURES if "_dedupe_" in n and
                                          n != "elb_rand_grain_content_key")


def call_form(native, name, shift, pct, dedupe_pct):
    """calls the entry point with len 0 / no descriptors; no call may launch a kernel"""
    before = native.elb_num_kernel_launches()
    res = getattr(native, name)(*DEDUPE_FORMS[name](shift, pct, dedupe_pct))
    assert native.elb_num_kernel_launches() == before
    return res


@pytest.mark.parametrize("name", sorted(DEDUPE_FORMS))
@pytest.mark.parametrize("shift,pct,dedupe_pct,message", [
    (12, 50, 101, "Dedupe percent must be in range 0..100. Given: 101"),
    (12, 101, 101, "Block variance percent must be in range 0..100. Given: 101"),
    (11, 50, 101, "Random verify grain shift must be in range 12..30. Given: 11"),
])
def test_content_argument_rejected_first(native, name, shift, pct, dedupe_pct, message):
    """checked in the order grain shift, pct, dedupe pct, before anything else"""
    assert call_form(native, name, shift, pct, dedupe_pct) == -1
    assert _native.last_error() == message


@pytest.mark.parametrize("name", sorted(n for n in DEDUPE_FORMS if n != "elb_verify_dedupe_grain"))
@pytest.mark.parametrize("shift,pct,dedupe_pct", [(12, 50, 100), (30, 0, 0), (20, 100, 1)])
def test_nothing_to_do_returns_0_without_launch(native, name, shift, pct, dedupe_pct):
    """(a single-block verify of len 0 resets its result, as K6's does)"""
    assert call_form(native, name, shift, pct, dedupe_pct) == 0


# ---- config and command line -------------------------------------------------------------------

def base_cfg(tmp_path, **kwargs):
    cfg = dict(paths=[str(tmp_path / "f")], block_size=4096, file_size=MiB,
               integrity_check_salt=5, integrity_check_kind=kernels.VERIFY_RANDOM,
               block_variance_percent=100, verify_random_grain=64 * KiB, dedupe_percent=50)
    cfg.update(kwargs)
    return WorkerConfig(**cfg)


def test_cfg_field_fills_padding():
    import ctypes
    assert ctypes.sizeof(_native.Cfg) == _native.load().elb_cfg_struct_size() == 360
    assert _native.Cfg.dedupePercent.offset == 180
    assert _native.Cfg.gpuIDs.offset == 184


NEEDS_GRAIN = ("A dedupe percentage (--dedupepct) requires a random verify grain "
               "(--verifyrandgrain).")


@pytest.mark.parametrize("kwargs,message", [
    (dict(dedupe_percent=101), "Dedupe percent must be in range 0..100. Given: 101"),
    (dict(verify_random_grain=0), NEEDS_GRAIN),
    (dict(integrity_check_kind=kernels.VERIFY_PATTERN, verify_random_grain=0), NEEDS_GRAIN),
    (dict(integrity_check_salt=0, verify_random_grain=0), NEEDS_GRAIN),
])
def test_config_rejections(tmp_path, kwargs, message):
    with pytest.raises(WorkerError) as excinfo:
        WorkerManager(base_cfg(tmp_path, **kwargs))
    assert str(excinfo.value) == message


def test_help_lists_the_option():
    for flag in ("--help-all", "--help"):
        res = run_cli(flag)
        assert res.returncode == 0
        text = " ".join(res.stdout.split())
        assert "--dedupepct" in text
        assert "Percentage of duplicate grains (0..100) in --verifyrandgrain data" in text


CLI = ["-w", "-s", "1g", "--gpuids", "0"]


@pytest.mark.parametrize("args,message", [
    (CLI + ["--dedupepct", "50", "/tmp/x"], 'Option "--dedupepct" requires "--verifyrandgrain"'),
    (CLI + ["--verifyrand", "2", "--dedupepct", "50", "/tmp/x"],
     'Option "--dedupepct" requires "--verifyrandgrain"'),
    (CLI + ["--verify", "2", "--dedupepct", "50", "/tmp/x"],
     'Option "--dedupepct" requires "--verifyrandgrain"'),
    (CLI + ["--verifyrand", "2", "--verifyrandgrain", "64k", "--dedupepct", "101", "/tmp/x"],
     'Option "--dedupepct" must be in range 0..100'),
    (CLI + ["--verifyrand", "2", "--verifyrandgrain", "64k", "--dedupepct", "1000", "/tmp/x"],
     'Option "--dedupepct" must be in range 0..100'),
])
def test_validation_messages(args, message):
    res = run_cli(*args)
    assert res.returncode == 1
    assert message in res.stderr, res.stderr


@pytest.mark.parametrize("args", [
    ["-w", "-r", "-b", "1M", "-s", "16M", "--verifyrand", "7", "--verifyrandgrain", "64K",
     "--dedupepct", "50"],
    ["-r", "-b", "4K", "-s", "16M", "--verifyrand", "7", "--verifyrandgrain", "4K",
     "--dedupepct", "100", "--rand", "--norandalign"],
    ["-w", "-b", "1M", "-s", "16M", "--verifyrand", "7", "--verifyrandgrain", "1M",
     "--dedupepct", "0"],
    ["-w", "-b", "1M", "-s", "16M", "--dedupepct", "0"],
])
def test_accepted_combinations(args):
    res = run_cli("--dryrun", *args, "--gpuids", "0", "/tmp/elb_dry_dedupe")
    assert res.returncode == 0, res.stderr


def test_dedupe_percent_travels_to_services(tmp_path):
    svc = FakeService(8 * MiB, [1000, 2000]).start()
    try:
        res = run_master("-w", "-r", "-t", "2", "-b", "1M", "-s", "8M", "--verifyrand", "77",
                         "--verifyrandgrain", "64K", "--dedupepct", "40", "--gpuids", "0",
                         "--hosts", "127.0.0.1:%d" % svc.port, "--nolive", str(tmp_path / "bench"))
        assert res.returncode == 0, res.stdout + res.stderr
        prep = svc.prepare_trees[0]
        assert prep["b200_dedupepct"] == "40"
        assert prep["b200_verifyrandgrain"] == str(64 * KiB)
    finally:
        svc.stop()
    plain = FakeService(8 * MiB, [1000, 2000]).start()
    try:
        res = run_master("-w", "-t", "2", "-b", "1M", "-s", "8M", "--verifyrand", "77",
                         "--verifyrandgrain", "64K", "--gpuids", "0", "--hosts",
                         "127.0.0.1:%d" % plain.port, "--nolive", str(tmp_path / "bench"))
        assert res.returncode == 0, res.stdout + res.stderr
        assert plain.prepare_trees[0]["b200_dedupepct"] == "0"
    finally:
        plain.stop()
