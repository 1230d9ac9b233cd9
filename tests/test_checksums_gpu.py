"""GPU tests of --checksums: the CRC kernel against the model (tests/crc_model.py) for ragged
windows, odd addresses and offsets, every length class and one block past 4 GiB; the worker end to
end (every complete line is zlib.crc32 of the file) in file, dir and custom tree mode over both
staging engines, AIO, --direct and cuFile, with and without block content; the rules of a phase
(any block size, thread count and queue depth give the same line, a flipped byte changes it, a
time-limited read is incomplete); an unchanged clean path; and the command line."""
import errno
import os
import random
import shutil
import subprocess
import tempfile
import zlib

import numpy as np
import pytest
import torch

MOCK_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mock_cufile")
# must be set before the native library binds cuFile for the first time in this process
os.environ.setdefault("ELB_CUFILE_LIB", os.path.join(MOCK_DIR, "libmock_cufile.so"))

from elbencho_b200 import BenchPhase, WorkerConfig, WorkerManager  # noqa: E402
from elbencho_b200 import kernels  # noqa: E402
from elbencho_b200.build import CLI_PATH  # noqa: E402
from elbencho_b200.worker import IOEngine, PathType  # noqa: E402
from tests import crc_model as model  # noqa: E402
from tests.test_custom_tree_gpu import TREE_TEXT  # noqa: E402

pytestmark = pytest.mark.gpu

KiB, MiB, GiB = 1 << 10, 1 << 20, 1 << 30
SEED = 0xC5C5


# ------------------------------------------------------------------------------------------------
# kernel level
# ------------------------------------------------------------------------------------------------

def raw_crc_of(data):
    """R(data) via zlib (the model's finish step undone)"""
    return zlib.crc32(data) ^ model.shift(0xFFFFFFFF, len(data)) ^ 0xFFFFFFFF


def run_kernel(blocks, publish):
    """blocks: [(device address, length, file offset, shift)] -> the launch's contributions"""
    stream = torch.cuda.current_stream().cuda_stream
    n = len(blocks)
    raw = kernels.pack_block_descs([(ptr, length, off, 0) for ptr, length, off, _ in blocks])
    descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).pin_memory()
    shifts = torch.tensor([s for *_, s in blocks], dtype=torch.int64).pin_memory()
    dev_crcs = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
    host_crcs = torch.full((max(n, 1),), 0x7777, dtype=torch.int32).pin_memory()
    ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
    before = kernels.num_kernel_launches()
    kernels.crc32_blocks(descs.data_ptr(), shifts.data_ptr(), n, dev_crcs.data_ptr(),
                         host_crcs.data_ptr() if publish else 0,
                         ticket.data_ptr() if publish else 0, stream)
    torch.cuda.synchronize()
    assert kernels.num_kernel_launches() == before + (1 if n else 0)
    if not publish:
        return [int(v) & 0xFFFFFFFF for v in dev_crcs.cpu().tolist()[:n]]
    assert int(ticket.item()) == 0  # re-armed
    assert not dev_crcs.any()       # zeroed for the next launch
    return [int(v) & 0xFFFFFFFF for v in host_crcs.tolist()[:n]]


def expected(buf, blocks, base_ptr):
    host = buf.cpu().numpy().tobytes()
    return [model.shift(raw_crc_of(host[ptr - base_ptr:ptr - base_ptr + length]), shift)
            for ptr, length, _, shift in blocks]


LENGTHS = [0, 1, 15, 16, 17, 4095, 4 * KiB, MiB]


@pytest.mark.parametrize("publish", [False, True])
@pytest.mark.parametrize("misalign", [0, 1, 3, 15])
def test_kernel_length_classes(cuda_device, misalign, publish):
    rng = random.Random(misalign)
    buf = torch.randint(0, 256, (len(LENGTHS) * (MiB + 64),), dtype=torch.uint8, device="cuda")
    blocks = []
    for i, length in enumerate(LENGTHS):
        ptr = buf.data_ptr() + i * (MiB + 64) + misalign
        blocks.append((ptr, length, rng.randrange(1 << 40) | 1, rng.choice(
            [0, 1, 7, rng.randrange(1 << 20), rng.randrange(1 << 33, 1 << 45)])))
    assert run_kernel(blocks, publish) == expected(buf, blocks, buf.data_ptr())


@pytest.mark.parametrize("seed,num_blocks,max_len", [
    (1, 1, 3 * MiB), (2, 7, 200 * KiB), (3, 64, 40 * KiB), (4, 300, 9000), (5, 2000, 4 * KiB),
    (6, 96, MiB),  # more 4 KiB chunks than the resident grid has warps: warps walk several
])
def test_kernel_ragged_windows(cuda_device, seed, num_blocks, max_len):
    rng = random.Random(seed)
    lengths = [rng.choice([0, 1, rng.randint(0, max_len), max_len]) for _ in range(num_blocks)]
    slot = max_len + 32
    buf = torch.randint(0, 256, (num_blocks * slot,), dtype=torch.uint8, device="cuda",
                        generator=torch.Generator("cuda").manual_seed(seed))
    blocks = [(buf.data_ptr() + i * slot + rng.randrange(16), length, rng.randrange(1 << 36),
               rng.randrange(1 << 40)) for i, length in enumerate(lengths)]
    assert run_kernel(blocks, True) == expected(buf, blocks, buf.data_ptr())


def test_kernel_window_is_a_file(cuda_device):
    """the blocks of a file in random order, with shift = bytes to the file end: their XOR
    finishes to zlib.crc32 of the file"""
    rng = random.Random(11)
    size = 3 * MiB + 12345
    buf = torch.randint(0, 256, (size,), dtype=torch.uint8, device="cuda")
    parts = model.random_split(size, rng)
    blocks = [(buf.data_ptr() + off, length, off, size - off - length) for off, length in parts]
    raw = 0
    for crc in run_kernel(blocks, True):
        raw ^= crc
    assert kernels.crc32_finish(raw, size) == zlib.crc32(buf.cpu().numpy().tobytes())


def test_kernel_block_past_4gib(cuda_device):
    length = 4 * GiB + 4099
    buf = torch.empty(length + 16, dtype=torch.uint8, device="cuda")
    buf.random_(0, 256, generator=torch.Generator("cuda").manual_seed(5))
    ptr = buf.data_ptr() + 5
    (crc,) = run_kernel([(ptr, length, 0, 0)], True)
    host = buf[5:5 + length].cpu().numpy()
    assert kernels.crc32_finish(crc, length) == zlib.crc32(host)
    del buf


# ------------------------------------------------------------------------------------------------
# worker level
# ------------------------------------------------------------------------------------------------

def can_open_direct(path):
    probe = os.path.join(path, ".direct_probe")
    try:
        os.close(os.open(probe, os.O_CREAT | os.O_RDWR | os.O_DIRECT, 0o600))
        return True
    except OSError as e:
        if e.errno == errno.EINVAL:
            return False
        raise
    finally:
        if os.path.exists(probe):
            os.unlink(probe)


def make_workdir(direct=False):
    base = "/dev/shm" if os.path.isdir("/dev/shm") and not direct else None
    path = tempfile.mkdtemp(prefix="elb_checksums_", dir=base)
    if direct and not can_open_direct(path):
        shutil.rmtree(path)
        pytest.skip("no O_DIRECT support under " + os.path.dirname(path))
    return path


@pytest.fixture()
def workdir(cuda_device):
    path = make_workdir()
    yield path
    shutil.rmtree(path, ignore_errors=True)


ENGINES = {
    "kernel": dict(staging_engine=1),
    "copyengine": dict(staging_engine=2),
    "aio": dict(io_engine=IOEngine.AIO, io_depth=8),
    "direct": dict(use_direct_io=True),
    "cufile": dict(use_cufile=True),
}

CONTENTS = {
    "verify": dict(integrity_check_salt=SEED),
    "grain": dict(integrity_check_salt=SEED, integrity_check_kind=kernels.VERIFY_RANDOM,
                  verify_random_grain=64 * KiB, block_variance_percent=100),
    "blockvar": dict(block_variance_percent=100),
    "none": dict(),
}


def setup_mode(mode, workdir, threads, whole_blocks):
    """-> (WorkerConfig arguments of the mode, {path: size} of its data set)"""
    if mode in ("file1", "file3"):
        paths = [os.path.join(workdir, "f%d" % i) for i in range(1 if mode == "file1" else 3)]
        # (--direct and --cufile round the data set size down to whole blocks: no 64 KiB tail)
        size = 6 * MiB + (0 if whole_blocks else 64 * KiB)
        return dict(paths=paths, file_size=size, block_size=256 * KiB), \
            {p: size for p in paths}
    if mode == "dir":
        size = 640 * KiB
        files = {os.path.join(workdir, "r%d" % r, "d%d" % d, "r%d-f%d" % (r, f)): size
                 for r in range(threads) for d in range(2) for f in range(2)}
        return dict(paths=[workdir], path_type=PathType.DIR, num_dirs=2, num_files=2,
                    file_size=size, block_size=128 * KiB), files
    tree_path = os.path.join(workdir, "tree.txt")
    bench_dir = os.path.join(workdir, "bench")
    os.mkdir(bench_dir)
    with open(tree_path, "w") as f:
        f.write(TREE_TEXT)
    files = {}
    for line in TREE_TEXT.splitlines():
        if line.startswith("f "):
            _, size, rel = line.split(" ", 2)
            files[os.path.join(bench_dir, rel)] = (int(size) + 4095) // 4096 * 4096
    return dict(paths=[bench_dir], path_type=PathType.DIR, tree_file_path=tree_path,
                tree_round_up_size=4096, block_size=64 * KiB, file_share_size=256 * KiB), files


def file_crc(path, size):
    with open(path, "rb") as f:
        data = f.read(size)
    assert len(data) == size, path
    return zlib.crc32(data)


def check_complete(lines, files):
    """every file of the data set is listed once, moved completely, with its zlib CRC"""
    assert [line[0] for line in lines] == sorted(files)
    for path, size, covered, crc in lines:
        assert size == files[path], path
        assert covered == size, path
        assert crc == file_crc(path, size), path


def run_phases(cfg, *phases):
    """-> the checksum lines of each phase"""
    sections = []
    with WorkerManager(cfg) as mgr:
        for phase in phases:
            mgr.run_phase(phase)
            if phase in (BenchPhase.CREATEFILES, BenchPhase.READFILES):
                sections.append(mgr.checksums())
    return sections


# (custom tree mode does not take --verifyrand data)
@pytest.mark.parametrize("mode,engine,content", [
    (mode, engine, content) for mode in ("file1", "file3", "dir", "tree") for engine in ENGINES
    for content in CONTENTS if (mode, content) != ("tree", "grain")])
def test_worker_lines_are_zlib_crcs(cuda_device, mode, engine, content):
    workdir = make_workdir(direct=(engine == "direct"))
    try:
        threads = 16 if mode.startswith("file") else 3
        args, files = setup_mode(mode, workdir, threads, engine in ("direct", "cufile"))
        if mode == "tree" and engine == "direct":
            args["no_direct_io_check"] = True
        cfg = WorkerConfig(num_threads=threads, checksums=True, **args, **ENGINES[engine],
                           **CONTENTS[content])
        phases = [BenchPhase.CREATEDIRS] if args.get("path_type") == PathType.DIR else []
        written, read = run_phases(cfg, *phases, BenchPhase.CREATEFILES, BenchPhase.READFILES)
        check_complete(written, files)
        assert read == written
    finally:
        shutil.rmtree(workdir, ignore_errors=True)


def test_lines_do_not_depend_on_block_size_threads_or_queue_depth(workdir):
    path = os.path.join(workdir, "f")
    size = 16 * MiB + 4 * KiB
    common = dict(paths=[path], file_size=size, checksums=True, block_variance_percent=100)
    (written,) = run_phases(WorkerConfig(block_size=MiB, num_threads=16, **common),
                            BenchPhase.CREATEFILES)
    (read,) = run_phases(WorkerConfig(block_size=4 * KiB, num_threads=3, io_depth=64,
                                      io_engine=IOEngine.AIO, **common), BenchPhase.READFILES)
    assert read == written == [(path, size, size, file_crc(path, size))]


def test_read_of_foreign_data(workdir):
    """a file that Python wrote, only read"""
    path = os.path.join(workdir, "f")
    data = np.random.default_rng(3).integers(0, 256, 5 * MiB + 3, dtype=np.uint8).tobytes()
    with open(path, "wb") as f:
        f.write(data)
    cfg = WorkerConfig(paths=[path], file_size=len(data), block_size=MiB, num_threads=4,
                       checksums=True)
    (read,) = run_phases(cfg, BenchPhase.READFILES)
    assert read == [(path, len(data), len(data), zlib.crc32(data))]


def test_flipped_byte_changes_the_read_line(workdir):
    path = os.path.join(workdir, "f")
    size = 4 * MiB
    cfg = WorkerConfig(paths=[path], file_size=size, block_size=MiB, num_threads=2,
                       checksums=True, block_variance_percent=100)
    written, clean = run_phases(cfg, BenchPhase.CREATEFILES, BenchPhase.READFILES)
    assert clean == written
    with open(path, "r+b") as f:
        f.seek(3 * MiB + 17)
        byte = f.read(1)
        f.seek(3 * MiB + 17)
        f.write(bytes([byte[0] ^ 0x20]))
    (damaged,) = run_phases(cfg, BenchPhase.READFILES)
    assert damaged[0][:3] == written[0][:3]
    assert damaged[0][3] != written[0][3]
    assert damaged[0][3] == file_crc(path, size)


def test_clean_path_costs_nothing(workdir):
    """without --checksums a phase launches and copies what it did before: one fill / verify
    launch per batch, the data once each way; with it, one CRC launch per batch more and no
    copy"""
    path = os.path.join(workdir, "f")
    size, block, batch_blocks = 8 * MiB, MiB, 2
    num_batches = size // block // batch_blocks
    counters = {}
    for checksums in (False, True):
        cfg = WorkerConfig(paths=[path], file_size=size, block_size=block,
                           pipeline_batch_blocks=batch_blocks, integrity_check_salt=SEED,
                           staging_engine=2, checksums=checksums)
        with WorkerManager(cfg) as mgr:
            for phase in (BenchPhase.CREATEFILES, BenchPhase.READFILES):
                r = mgr.run_phase(phase)
                counters[checksums, phase] = (r["num_kernel_launches"], r["h2d_bytes"],
                                              r["d2h_bytes"])
    assert counters[False, BenchPhase.CREATEFILES] == (num_batches, 0, size)
    assert counters[False, BenchPhase.READFILES] == (num_batches, size, 0)
    assert counters[True, BenchPhase.CREATEFILES] == (2 * num_batches, 0, size)
    assert counters[True, BenchPhase.READFILES] == (2 * num_batches, size, 0)


# ------------------------------------------------------------------------------------------------
# command line
# ------------------------------------------------------------------------------------------------

def run_cli(*args):
    return subprocess.run([CLI_PATH] + list(args), capture_output=True, text=True, timeout=300)


def parse_sections(text):
    sections = []
    for line in text.splitlines():
        if line.startswith("# phase "):
            sections.append((line[len("# phase "):], []))
        else:
            path, size, covered, crc = line.rsplit(" ", 3)
            sections[-1][1].append((path, int(size), int(covered), crc))
    return sections


def test_cli_write_read(workdir):
    paths = [os.path.join(workdir, "a"), os.path.join(workdir, "b")]
    sums = os.path.join(workdir, "sums.txt")
    with open(sums, "w") as f:
        f.write("stale\n")
    size = 8 * MiB
    res = run_cli("-w", "-r", "-b", "1m", "-s", "8m", "-t", "4", "--verify", "7", "--gpuids", "0",
                  "--nolive", "--checksums", sums, *paths)
    assert res.returncode == 0, res.stderr
    assert res.stdout.count("Checksums: 2 files, 2 complete: %s\n" % sums) == 2
    with open(sums) as f:
        sections = parse_sections(f.read())
    want = [(p, size, size, "%08x" % file_crc(p, size)) for p in paths]
    assert sections == [("WRITE", want), ("READ", want)]


def test_cli_time_limited_read_is_incomplete(workdir):
    path = os.path.join(workdir, "f")
    sums = os.path.join(workdir, "sums.txt")
    common = ["-b", "64k", "-s", "64m", "-t", "2", "--gpuids", "0", "--nolive", "--checksums",
              sums, path]
    assert run_cli("-w", *common).returncode == 0
    res = run_cli("-r", "--timelimit", "1", "--limitread", "1m", *common)
    assert res.returncode == 0, res.stderr
    assert "Checksums: 1 files, 0 complete: %s\n" % sums in res.stdout
    with open(sums) as f:
        ((phase, [(got_path, size, covered, crc)]),) = parse_sections(f.read())
    assert (phase, got_path, size, crc) == ("READ", path, 64 * MiB, "-")
    assert 0 < covered < size and covered % (64 * KiB) == 0
