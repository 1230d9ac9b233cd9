"""CPU tests of --verifyrand: the closed forms that key each block's random data by its place in
the data set (library export against the CPU restatement), the reference verify of random blocks,
the command line option with its rejections, the service key, and the unchanged elb_cfg layout."""
import ctypes
import random

import numpy as np
import pytest

from elbencho_b200 import WorkerConfig, WorkerError, WorkerManager, _native, kernels
from elbencho_b200.worker import PathType
from tests import kernel_cases as kc
from tests import verify_random_model as model
from tests.test_cli import run_cli
from tests.test_master_fake_services import FakeService, run_master

MiB = 1 << 20

# (fileKey, fileOffset) -> elb_rand_pos_counter
POS_COUNTER_KAT = [
    ((0, 0), 5197578548964807871),
    ((1, 4096), 167847659046587400),
    ((7, (1 << 63) + 5), 10168587252987297532),
    ((model.U64, model.U64), 5066756352113716771),
]
# (rank, dirIndex, fileIndex) -> elb_rand_dir_file_key
DIR_FILE_KEY_KAT = [
    ((0, 0, 0), 0),
    ((3, 1, 2), 4368362667439261810),
    ((127, 63, 127), 4834859165808419607),
]


@pytest.mark.parametrize("args,want", POS_COUNTER_KAT)
def test_pos_counter_known_answers(args, want):
    assert kernels.rand_pos_counter(*args) == want
    assert model.pos_counter(*args) == want


@pytest.mark.parametrize("args,want", DIR_FILE_KEY_KAT)
def test_dir_file_key_known_answers(args, want):
    assert kernels.rand_dir_file_key(*args) == want
    assert model.dir_file_key(*args) == want


def test_closed_forms_agree_on_seeded_inputs():
    rng = random.Random(5)
    for _ in range(200):
        key, off = rng.getrandbits(64), rng.getrandbits(64)
        assert kernels.rand_pos_counter(key, off) == model.pos_counter(key, off)
        r, d, f = rng.getrandbits(20), rng.getrandbits(20), rng.getrandbits(20)
        assert kernels.rand_dir_file_key(r, d, f) == model.dir_file_key(r, d, f)


def test_pos_counters_of_a_file_are_distinct():
    """one file's blocks never share a key; files with different keys differ at the same offset"""
    block = 4096
    for key in (0, 1, model.dir_file_key(2, 0, 1)):
        ctrs = {model.pos_counter(key, off) for off in range(0, 4096 * block, block)}
        assert len(ctrs) == 4096
    assert model.pos_counter(0, 0) != model.pos_counter(1, 0)
    # the dir mode key tells the three numbers apart in any order
    keys = {model.dir_file_key(*t) for t in [(1, 2, 3), (1, 3, 2), (2, 1, 3), (2, 3, 1),
                                             (3, 1, 2), (3, 2, 1)]}
    assert len(keys) == 6


@pytest.mark.parametrize("pct", kc.PCTS)
def test_reference_verify_agrees_with_numpy(pct):
    """the oracle-backed verify against a numpy restatement: odd lengths, flips at the head, on
    both sides of the var/const boundary and at the tail"""
    rng = random.Random(pct)
    for length in (1, 7, 17, 255, 4097, 65536 + 13):
        seed, ctr = rng.getrandbits(64), rng.getrandbits(64)
        want = kc.random_bytes(length, pct, seed, ctr, 0, length)
        base = model.random_block(length, pct, seed, ctr)
        assert np.array_equal(base, want)
        assert model.verify_random(base.tobytes(), pct, seed, ctr) == (0, model.U64)
        var_len = kc.rand_var_fill_len(length, pct)
        flips = sorted({p for p in (0, var_len - 1, var_len, length - 1) if 0 <= p < length})
        data = bytearray(base.tobytes())
        for p in flips:
            data[p] ^= 0x5A
        bad = np.flatnonzero(np.frombuffer(bytes(data), dtype=np.uint8) != want)
        assert model.verify_random(data, pct, seed, ctr) == (len(flips), flips[0])
        assert list(bad) == flips
        # another seed: almost every byte differs
        count, first = model.verify_random(base.tobytes(), pct, seed ^ 1, ctr)
        assert count == int(np.count_nonzero(
            kc.random_bytes(length, pct, seed ^ 1, ctr, 0, length) != want))


def test_file_content_and_error_text_model():
    size, block, pct, seed = 3 * 4096 + 100, 4096, 100, 99
    data = bytearray(model.file_random_content(size, block, pct, seed, 0))
    assert model.error_text(bytes(data), block, pct, seed, 0) is None
    data[5000] ^= 1
    want = model.random_block(4096, pct, seed, model.pos_counter(0, 4096))[5000 - 4096]
    assert model.error_text(bytes(data), block, pct, seed, 0) == (
        "Data verification failed. Offset: 5000; Expected value: %d; Actual value: %d"
        % (want, want ^ 1))


# ---- C ABI -------------------------------------------------------------------------------------

def test_cfg_layout_is_unchanged():
    """integrityCheckKind took the place of a reserved int32: size and ABI version stay"""
    lib = _native.load()
    assert lib.elb_cfg_struct_size() == ctypes.sizeof(_native.Cfg) == 360
    assert lib.elb_abi_version() == 1
    fields = [f[0] for f in _native.Cfg._fields_]
    assert fields[-1] == "integrityCheckKind"
    assert _native.Cfg.integrityCheckKind.offset == _native.Cfg.useNoFDSharing.offset + 4


@pytest.mark.parametrize("kwargs,message", [
    (dict(integrity_check_kind=2), "Invalid integrity check kind: 2"),
    (dict(rwmix_read_percent=10), "Integrity check cannot be used together with rwmixpct."),
    (dict(use_random_offsets=True, use_random_unaligned=True, rand_offset_seed=1),
     "Random data verification (--verifyrand) cannot be used together with unaligned random "
     "offsets."),
])
def test_config_rejections(tmp_path, kwargs, message):
    cfg = dict(paths=[str(tmp_path / "f")], block_size=4096, file_size=MiB,
               integrity_check_salt=5, integrity_check_kind=kernels.VERIFY_RANDOM,
               block_variance_percent=100)
    cfg.update(kwargs)
    with pytest.raises(WorkerError) as excinfo:
        WorkerManager(WorkerConfig(**cfg))
    assert str(excinfo.value) == message


def test_config_rejects_custom_tree(tmp_path):
    tree = tmp_path / "tree.txt"
    tree.write_text("d d1\nf 4096 d1/a\n")
    cfg = WorkerConfig(paths=[str(tmp_path)], path_type=PathType.DIR, block_size=4096,
                       file_size=4096, integrity_check_salt=5,
                       integrity_check_kind=kernels.VERIFY_RANDOM, tree_file_path=str(tree))
    with pytest.raises(WorkerError) as excinfo:
        WorkerManager(cfg)
    assert str(excinfo.value) == "Custom tree mode cannot be used together with --verifyrand."


# ---- command line ------------------------------------------------------------------------------

def test_help_describes_the_option():
    res = run_cli("--help")
    assert res.returncode == 0
    text = " ".join(res.stdout.split())
    assert "--verifyrand" in text
    assert "not block size independent" in text and "[b200]" in text


@pytest.mark.parametrize("args,message", [
    (["-w", "-s", "1g", "--gpuids", "0", "--verify", "1", "--verifyrand", "2", "/tmp/x"],
     'Option "--verifyrand" cannot be used together with "--verify"'),
    (["-w", "-s", "1g", "--gpuids", "0", "--verifyrand", "2", "--rwmixpct", "10", "/tmp/x"],
     'Option --rwmixpct cannot be used together with option "--verifyrand"'),
    (["-w", "-s", "1g", "--gpuids", "0", "--rand", "--verifyrand", "2", "/tmp/x"],
     "Integrity check writes are not supported in combination with random offsets."),
    (["-w", "-s", "1g", "--gpuids", "0", "--verifyrand", "2", "--treefile", "/tmp/t.txt",
      "/tmp"], "Custom tree mode cannot be used together with --verifyrand."),
    (["-r", "-s", "1g", "--gpuids", "0", "--verifyrand", "2", "--verifydirect", "/tmp/x"],
     "Direct verification requires --verify and --write"),
    (["-w", "-s", "1g", "--gpuids", "0", "--verifydirect", "/tmp/x"],
     "Direct verification requires --verify and --write"),
])
def test_validation_messages(args, message):
    res = run_cli(*args)
    assert res.returncode == 1
    assert message in res.stderr, res.stderr


@pytest.mark.parametrize("args", [
    ["-w", "-r", "-b", "1M", "-s", "8M", "--verifyrand", "7"],
    ["-w", "-b", "1M", "-s", "8M", "--verifyrand", "7", "--verifydirect"],
    ["-w", "-r", "-b", "1M", "-s", "8M", "--verifyrand", "7", "--blockvarpct", "40"],
    ["-r", "-b", "4K", "-s", "8M", "--verifyrand", "7", "--rand"],  # random reads are fine
])
def test_accepted_combinations(args):
    res = run_cli("--dryrun", *args, "--gpuids", "0", "/tmp/elb_dry_vr")
    assert res.returncode == 0, res.stderr


def test_seed_travels_to_services(tmp_path):
    svc = FakeService(8 * MiB, [1000, 2000]).start()
    try:
        res = run_master("-w", "-r", "-t", "2", "-b", "1M", "-s", "8M", "--verifyrand", "77",
                         "--gpuids", "0", "--hosts", "127.0.0.1:%d" % svc.port, "--nolive",
                         str(tmp_path / "bench"))
        assert res.returncode == 0, res.stdout + res.stderr
        prep = svc.prepare_trees[0]
        assert prep["b200_verifyrand"] == "77"
        assert prep["verify"] == "0"
    finally:
        svc.stop()
    plain = FakeService(8 * MiB, [1000, 2000]).start()
    try:
        res = run_master("-w", "-t", "2", "-b", "1M", "-s", "8M", "--gpuids", "0", "--hosts",
                         "127.0.0.1:%d" % plain.port, "--nolive", str(tmp_path / "bench"))
        assert res.returncode == 0, res.stdout + res.stderr
        assert plain.prepare_trees[0]["b200_verifyrand"] == "0"
    finally:
        plain.stop()
