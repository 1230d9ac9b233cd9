"""GPU tests of --verifyreport: the damage map kernel against the model for all four contents and
every block shape, the worker end to end (the report equals the model of tests/
verify_report_model.py over both staging engines, sync and AIO, 1 and 4 threads, 4 KiB and 1 MiB
blocks, sequential and random offsets, dir mode and cuFile), the phase-level rules (every byte
read, the error text, the byte sum, an unchanged clean read) and the command line."""
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

MOCK_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mock_cufile")
# must be set before the native library binds cuFile for the first time in this process
os.environ.setdefault("ELB_CUFILE_LIB", os.path.join(MOCK_DIR, "libmock_cufile.so"))

from elbencho_b200 import BenchPhase, WorkerConfig, WorkerError, WorkerManager  # noqa: E402
from elbencho_b200 import _native, kernels  # noqa: E402
from elbencho_b200.build import CLI_PATH  # noqa: E402
from elbencho_b200.worker import IOEngine, PathType  # noqa: E402
from tests import verify_random_model as vrm  # noqa: E402
from tests import verify_report_model as model  # noqa: E402

pytestmark = pytest.mark.gpu

KiB, MiB = 1 << 10, 1 << 20
SEED = 0x5EC7
SHIFT = 14  # 16 KiB grains


# ------------------------------------------------------------------------------------------------
# kernel level
# ------------------------------------------------------------------------------------------------

CONTENTS = ["pattern", "random", "grain", "dedupe"]


def fill(content, ptr, length, file_offset, key, stream):
    if content == "pattern":
        kernels.fill_pattern(ptr, length, file_offset, SEED, stream)
    elif content == "random":
        kernels.fill_random(ptr, length, 70, SEED, key, stream)
    elif content == "grain":
        kernels.fill_random_grain(ptr, length, file_offset, SHIFT, 70, SEED, key, stream)
    else:
        kernels.fill_dedupe_grain(ptr, length, file_offset, SHIFT, 70, 40, SEED, key, stream)


def content_args(content):
    """(contentKind, key, pct, grainShift, dedupePct) of elb_damage_map"""
    return {"pattern": (kernels.CONTENT_PATTERN, SEED, 0, 0, 0),
            "random": (kernels.CONTENT_RANDOM, SEED, 70, 0, 0),
            "grain": (kernels.CONTENT_RANDOM_GRAIN, SEED, 70, SHIFT, 0),
            "dedupe": (kernels.CONTENT_RANDOM_GRAIN, SEED, 70, SHIFT, 40)}[content]


# (name, device misalignment, length, file offset, damaged block positions)
SHAPES = [
    ("one byte", 0, 64 * KiB, 1 << 20, [777]),
    ("run across a sector boundary", 0, 64 * KiB, 1 << 20, list(range(500, 530))),
    ("whole block", 0, 8 * KiB, 3 << 20, list(range(8 * KiB))),
    ("unaligned file offset", 0, 40 * KiB + 5, (1 << 20) + 1234, [0, 1, 300, 5000, 40 * KiB + 4]),
    ("unaligned device address", 3, 32 * KiB, 1 << 20, [0, 511, 512, 20000, 32 * KiB - 1]),
    ("shorter than a sector", 0, 300, 4096 + 100, [0, 150, 299]),
    ("shorter than a sector, across one", 7, 300, 4096 + 400, [0, 111, 112, 299]),
    ("not a multiple of 512", 0, 4096 + 700, 8192, [4096, 4096 + 699, 4200]),
    ("head and tail of a long block", 5, (1 << 20) + 333, (5 << 20) + 17,
     [0, 1, 2, 15, 16, (1 << 20) + 332, (1 << 20) + 320]),
]


def records_of(sectors, count):
    raw = sectors.cpu().numpy().reshape(-1, 4)[:count]
    return [(int(n), int(f), int(la)) for n, f, la, _ in raw]


@pytest.mark.parametrize("content", CONTENTS)
@pytest.mark.parametrize("shape", SHAPES, ids=[s[0] for s in SHAPES])
def test_kernel_against_model(cuda_device, content, shape):
    _, misalign, length, file_offset, damage = shape
    stream = torch.cuda.current_stream().cuda_stream
    key = 12345
    buf = torch.zeros(length + 64, dtype=torch.uint8, device="cuda")
    ptr = buf.data_ptr() + misalign
    fill(content, ptr, length, file_offset, key, stream)
    torch.cuda.synchronize()
    clean = buf[misalign:misalign + length].cpu().numpy().copy()
    idx = torch.tensor(damage, dtype=torch.long, device="cuda") + misalign
    buf[idx] ^= 0x41
    torch.cuda.synchronize()
    dirty = buf[misalign:misalign + length].cpu().numpy().copy()

    first_sector = file_offset // 512
    num_sectors = (file_offset + length - 1) // 512 - first_sector + 1
    per_desc = num_sectors + 3
    descs = torch.frombuffer(bytearray(kernels.pack_block_descs([(ptr, length, file_offset, key)])),
                             dtype=torch.uint8).pin_memory()
    sectors = torch.full((per_desc * 4,), 0x7777, dtype=torch.int32, device="cuda")
    before = kernels.num_kernel_launches()
    kernels.damage_map(descs.data_ptr(), 1, *content_args(content), sectors.data_ptr(), per_desc,
                       stream)
    torch.cuda.synchronize()
    assert kernels.num_kernel_launches() == before + 1
    got = records_of(sectors, per_desc)

    # the model, on file positions
    pad = bytes(file_offset)
    recs = model.sector_records(pad + clean.tobytes(), pad + dirty.tobytes(),
                                [(file_offset, length)])
    want = [(0, 0, 0)] * num_sectors
    for sector, _, count, first, last in recs:
        want[sector - first_sector] = (count, first % 512, last % 512)
    assert got[:num_sectors] == want
    assert got[num_sectors:] == [(0x7777, 0x7777, 0x7777)] * 3  # records past the block untouched


def test_kernel_many_descriptors(cuda_device):
    """a batch of bad blocks of different lengths and offsets, one launch"""
    stream = torch.cuda.current_stream().cuda_stream
    blocks, cleans, dirties, slot = [], [], [], 1 << 20
    buf = torch.zeros(8 * slot, dtype=torch.uint8, device="cuda")
    rng = np.random.default_rng(7)
    for i in range(8):
        length = int(rng.integers(1, slot - 600))
        off = int(rng.integers(0, 1 << 30))
        ptr = buf.data_ptr() + i * slot
        fill("grain", ptr, length, off, i, stream)
        blocks.append((ptr, length, off, i))
    torch.cuda.synchronize()
    for i, (ptr, length, off, key) in enumerate(blocks):
        cleans.append(buf[i * slot:i * slot + length].cpu().numpy().copy())
        pos = rng.integers(0, length, size=50)
        buf[torch.tensor(pos + i * slot, device="cuda")] ^= 0x10
    torch.cuda.synchronize()
    for i, (ptr, length, off, key) in enumerate(blocks):
        dirties.append(buf[i * slot:i * slot + length].cpu().numpy().copy())
    per_desc = slot // 512 + 2
    descs = torch.frombuffer(bytearray(kernels.pack_block_descs(blocks)),
                             dtype=torch.uint8).pin_memory()
    sectors = torch.zeros(8 * per_desc * 4, dtype=torch.int32, device="cuda")
    kernels.damage_map(descs.data_ptr(), 8, *content_args("grain"), sectors.data_ptr(), per_desc,
                       stream)
    torch.cuda.synchronize()
    raw = sectors.cpu().numpy().reshape(8, per_desc, 4)
    for i, (ptr, length, off, key) in enumerate(blocks):
        # compare against the model in block-relative form (shift the file by off % 512)
        shift = off % 512
        pad = bytes(shift)
        recs = model.sector_records(pad + cleans[i].tobytes(), pad + dirties[i].tobytes(),
                                    [(shift, length)])
        num_sectors = (off + length - 1) // 512 - off // 512 + 1
        want = np.zeros((num_sectors, 3), dtype=np.int64)
        for sector, _, count, first, last in recs:
            want[sector] = (count, first % 512, last % 512)
        assert (raw[i, :num_sectors, :3] == want).all(), i


# ------------------------------------------------------------------------------------------------
# worker level
# ------------------------------------------------------------------------------------------------

@pytest.fixture(params=["kernel", "copyengine"])
def staging_engine(request, monkeypatch):
    monkeypatch.setenv("ELB_STAGING", request.param)
    return request.param


@pytest.fixture()
def workdir(cuda_device):
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    path = tempfile.mkdtemp(prefix="elb_vreport_", dir=base)
    yield path
    shutil.rmtree(path, ignore_errors=True)


SIZE = 8 * MiB


def cfg_of(paths, content, **kwargs):
    args = dict(paths=paths, block_size=MiB, file_size=SIZE, integrity_check_salt=SEED)
    if content != "pattern":
        args.update(integrity_check_kind=kernels.VERIFY_RANDOM, block_variance_percent=70)
    if content in ("grain", "dedupe"):
        args.update(verify_random_grain=1 << SHIFT)
    if content == "dedupe":
        args.update(dedupe_percent=40)
    args.update(kwargs)
    return WorkerConfig(**args)


def expected_content(content, size, file_key=0, block=MiB):
    if content == "pattern":
        return model.pattern_content(0, size, SEED)
    if content == "random":
        return model.block_random_content(size, block, 70, SEED, file_key)
    return model.grain_content(size, 1 << SHIFT, 70, SEED, file_key,
                               40 if content == "dedupe" else 0)


# damage in every quarter of the file (every worker's range with 4 threads), across sector,
# 4 KiB and 1 MiB boundaries, and a whole 4 KiB block
DAMAGE = [(0, b"\x01"), (4090, bytes(11)), (700, b"\xff" * 3), (2 * MiB - 2, b"\x00" * 5),
          (2 * MiB + 8192, b"\x13" * 4096), (5 * MiB + 511, b"\x77\x88"), (SIZE - 1, b"\x99")]


def damage(path, spots=DAMAGE):
    fd = os.open(path, os.O_RDWR)
    try:
        for off, data in spots:
            old = os.pread(fd, len(data), off)
            os.pwrite(fd, bytes(a ^ b ^ 0x5A for a, b in zip(old, data)), off)
    finally:
        os.close(fd)


def write(paths, content, **kwargs):
    with WorkerManager(cfg_of(paths, content, **kwargs)) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)


def read_with_report(cfg):
    """-> (error text or None, phase results, report lines)"""
    with WorkerManager(cfg) as mgr:
        mgr.start_phase(BenchPhase.READFILES)
        try:
            mgr.wait_done(-1)
            err = None
        except WorkerError as e:
            err = str(e)
        return err, mgr.phase_results(), mgr.verify_report()


def read_error(cfg):
    with WorkerManager(cfg) as mgr:
        with pytest.raises(WorkerError) as excinfo:
            mgr.run_phase(BenchPhase.READFILES)
        return str(excinfo.value)


def block_grid(size, block):
    return [(off, min(block, size - off)) for off in range(0, size, block)]


def file_model(path, content, ranges, block=MiB, file_key=0):
    with open(path, "rb") as f:
        actual = f.read()
    files = {path: (expected_content(content, len(actual), file_key, block), actual)}
    return model.extents(files, {path: ranges})


def check_full_read(path, content, block, threads, **kwargs):
    cfg = cfg_of([path], content, block_size=block, num_threads=threads, **kwargs)
    err, res, lines = read_with_report(cfg)
    want = file_model(path, content, block_grid(SIZE, block))
    assert lines == want
    assert res["ops_total"]["bytes"] == SIZE  # read on past the damage
    assert res["num_workers_done"] == threads
    assert sum(line[3] for line in lines) == res["verify_mismatch_bytes"]
    quarters = {line[1] * 4 // SIZE for line in lines}
    assert quarters == {0, 1, 2, 3}
    return err


@pytest.mark.parametrize("io", ["sync", "aio"])
@pytest.mark.parametrize("threads", [1, 4])
@pytest.mark.parametrize("block", [4 * KiB, MiB])
def test_worker_sequential(workdir, staging_engine, io, threads, block):
    path = os.path.join(workdir, "f")
    write([path], "pattern")
    damage(path)
    io_args = (dict(io_engine=IOEngine.SYNC) if io == "sync" else
               dict(io_engine=IOEngine.AIO, io_depth=4))
    err = check_full_read(path, "pattern", block, threads, verify_report=True, **io_args)
    # the error of the lowest-ranked worker that found damage: rank 0 reads the file's start
    plain = read_error(cfg_of([path], "pattern", block_size=block, num_threads=1, **io_args))
    assert err == plain
    assert plain.startswith("Data verification failed. Offset: 0; ")


@pytest.mark.parametrize("content", ["random", "grain", "dedupe"])
def test_worker_random_contents(workdir, staging_engine, content):
    path = os.path.join(workdir, "f")
    write([path], content)
    damage(path)
    err = check_full_read(path, content, MiB, 4, verify_report=True)
    assert err == read_error(cfg_of([path], content, num_threads=1))


def offset_plan_ranges(native, kind, amount, block, seed, rank=0):
    state = (ctypes.c_uint64 * 4)()
    native.elb_expand_offset_seed(seed, rank, state)
    plan = native.elb_offset_plan_create_algo(kind, amount, SIZE, 0, block, 1, 0, state,
                                              state[0] ^ state[1], 1)
    assert plan
    out, off, length = [], ctypes.c_uint64(), ctypes.c_uint64()
    try:
        while native.elb_offset_plan_next(plan, ctypes.byref(off), ctypes.byref(length)):
            out.append((off.value, length.value))
    finally:
        native.elb_offset_plan_destroy(plan)
    return out


@pytest.mark.parametrize("unaligned", [False, True])
def test_worker_random_offsets(workdir, staging_engine, native, unaligned):
    """random reads with replacement (--randamount twice the file): sectors read more than once
    count once; --norandalign reads grain data at unaligned offsets"""
    path = os.path.join(workdir, "f")
    write([path], "grain")
    damage(path)
    block = 4 * KiB
    kwargs = dict(block_size=block, num_threads=1, use_random_offsets=True,
                  use_random_unaligned=unaligned, random_amount=2 * SIZE, rand_offset_seed=99,
                  verify_report=True)
    err, res, lines = read_with_report(cfg_of([path], "grain", **kwargs))
    ranges = offset_plan_ranges(native, 2 if unaligned else 3, 2 * SIZE, block, 99)
    assert sum(n for _, n in ranges) == res["ops_total"]["bytes"] == 2 * SIZE
    assert lines == file_model(path, "grain", ranges)
    assert lines and err.startswith("Data verification failed. Offset: ")


def test_worker_dir_mode(workdir, staging_engine):
    cfg = dict(paths=[workdir], path_type=PathType.DIR, num_threads=2, num_dirs=1, num_files=2,
               file_size=SIZE // 4, block_size=64 * KiB)
    with WorkerManager(cfg_of(content="random", **cfg)) as mgr:
        mgr.run_phase(BenchPhase.CREATEDIRS)
        mgr.run_phase(BenchPhase.CREATEFILES)
    names = {}
    for rank in range(2):
        for fidx in range(2):
            path = os.path.join(workdir, "r%d" % rank, "d0", "r%d-f%d" % (rank, fidx))
            damage(path, [(100 + fidx, b"\x01"), (70000, b"\x02" * 1000)])
            names[path] = vrm.dir_file_key(rank, 0, fidx)
    err, res, lines = read_with_report(cfg_of(content="random", verify_report=True, **cfg))
    want = []
    for path, key in sorted(names.items()):
        want += file_model(path, "random", block_grid(SIZE // 4, 64 * KiB), 64 * KiB, key)
    assert lines == want
    assert res["ops_total"]["bytes"] == SIZE
    assert err.startswith("Data verification failed. Offset: 100; ")


def test_worker_cufile(workdir):
    path = os.path.join(workdir, "f")
    cfg = dict(block_size=512 * KiB, num_threads=2, use_cufile=True, use_gds_buf_reg=True,
               pipeline_batch_blocks=3)
    write([path], "grain", **cfg)
    damage(path)
    err, res, lines = read_with_report(cfg_of([path], "grain", verify_report=True, **cfg))
    assert lines == file_model(path, "grain", block_grid(SIZE, 512 * KiB))
    assert res["ops_total"]["bytes"] == SIZE
    assert err.startswith("Data verification failed. Offset: 0; ")


def test_verifydirect_and_collect_all(workdir, staging_engine):
    """a clean --verifydirect write reports nothing; with verifyCollectAll a damaged read has no
    error and still reports"""
    path = os.path.join(workdir, "f")
    with WorkerManager(cfg_of([path], "pattern", do_direct_verify=True, verify_report=True,
                              block_size=64 * KiB)) as mgr:
        w = mgr.run_phase(BenchPhase.CREATEFILES)
        assert w["verified_bytes"] == SIZE and mgr.verify_report() == []
    damage(path)
    err, res, lines = read_with_report(cfg_of([path], "pattern", verify_report=True,
                                              verify_collect_all=True, num_threads=4))
    assert err is None
    assert lines == file_model(path, "pattern", block_grid(SIZE, MiB))


def test_clean_read_costs_nothing(workdir, staging_engine):
    path = os.path.join(workdir, "f")
    write([path], "grain")
    counters = []
    for report in (False, True):
        with WorkerManager(cfg_of([path], "grain", num_threads=4, verify_report=report)) as mgr:
            r = mgr.run_phase(BenchPhase.READFILES)
            assert mgr.verify_report() == []
        counters.append((r["num_kernel_launches"], r["h2d_bytes"], r["d2h_bytes"],
                         r["verified_bytes"], r["verify_mismatch_bytes"]))
    assert counters[0] == counters[1]


# ------------------------------------------------------------------------------------------------
# command line
# ------------------------------------------------------------------------------------------------

def run_cli(*args):
    return subprocess.run([CLI_PATH] + list(args), capture_output=True, text=True, timeout=300)


def test_cli_report_file(workdir):
    path = os.path.join(workdir, "f")
    report = os.path.join(workdir, "report.txt")
    common = ["-b", "1m", "-s", "8m", "-t", "2", "--verify", str(SEED), "--gpuids", "0",
              "--nolive", "--verifyreport", report]
    res = run_cli("-w", "--verifydirect", *common, path)
    assert res.returncode == 0, res.stderr
    with open(report) as f:
        assert f.read() == "# phase WRITE\n"
    assert "Verify report: 0 damaged extents, 0 differing bytes in 0 files: %s\n" % report \
        in res.stdout
    damage(path)
    res = run_cli("-r", *common, path)
    assert res.returncode == 1
    lines = file_model(path, "pattern", block_grid(SIZE, MiB))
    with open(report) as f:  # truncated at start: only the read's section
        assert f.read() == "# phase READ\n" + model.report_text(lines)
    assert ("Verify report: %d damaged extents, %d differing bytes in 1 files: %s\n"
            % (len(lines), sum(line[3] for line in lines), report)) in res.stdout
    assert "ERROR: Data verification failed. Offset: 0; " in res.stderr
    plain = run_cli("-r", *common[:4], "-t", "1", *common[6:-2], path)
    assert plain.returncode == 1
    assert plain.stderr == res.stderr
