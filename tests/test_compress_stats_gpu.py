"""GPU tests of --compressstats: the LZ4 kernel's sizes and bytes against tests/compress_model.py
(every chunk size, ragged last chunks, odd device addresses, several descriptors, a block past
4 GiB), two streams into one counter block, the setter's rejections, then the worker's counts
against the model applied to the files on disk (block sizes, threads, AIO, staging engines,
--direct, mock cuFile, dir mode, custom tree mode), a random read of uniform data, the last data
set thread's remainder, two GPUs, the launches and copies with and without the option, and the
console line of the command line."""
import ctypes
import os
import shutil

import numpy as np
import pytest
import torch

from tests import test_checksums_gpu as base  # noqa: F401  (sets the mock cuFile library first)
from elbencho_b200 import BenchPhase, WorkerConfig, WorkerError, WorkerManager  # noqa: E402
from elbencho_b200 import _native, kernels  # noqa: E402
from elbencho_b200.worker import IOEngine, PathType  # noqa: E402
from tests import compress_model as model  # noqa: E402
from tests import tree_model  # noqa: E402
from tests.test_compress_stats import make_data  # noqa: E402
from tests.test_custom_tree_gpu import TREE_TEXT  # noqa: E402
from tests.test_checksums_gpu import make_workdir, run_cli  # noqa: E402

pytestmark = pytest.mark.gpu

KiB, MiB, GiB = 1 << 10, 1 << 20, 1 << 30


def _launch(blocks, shift, slots, counters, stream=None, with_bytes=True):
    """blocks: [(device tensor, byte offset in it, length, file offset)] -> (sizes, out) tensors"""
    raw = kernels.pack_block_descs([(t.data_ptr() + o, n, f, 0) for t, o, n, f in blocks])
    descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).pin_memory()
    sizes = torch.zeros(len(blocks) * slots, dtype=torch.int32, device="cuda")
    out = torch.zeros(len(blocks) * slots * kernels.lz4_out_slot_bytes(shift) if with_bytes else 1,
                      dtype=torch.uint8, device="cuda")
    s = stream or torch.cuda.current_stream()
    with torch.cuda.stream(s):
        kernels.lz4_chunks(descs.data_ptr(), len(blocks), shift, slots, counters.data_ptr(),
                           sizes.data_ptr(), out.data_ptr() if with_bytes else 0, s.cuda_stream)
    return descs, sizes, out


def _check_against_model(datas, shift, blocks, slots, sizes, out, with_bytes=True):
    chunk = 1 << shift
    slot_bytes = kernels.lz4_out_slot_bytes(shift)
    sizes = sizes.cpu().numpy().astype(np.int64)
    host = out.cpu().numpy() if with_bytes else None
    want_counts = [0, 0, 0, 0]
    for i, data in enumerate(datas):
        for j, o in enumerate(range(0, len(data), chunk)):
            piece = data[o:o + chunk]
            block = model.compress(piece)
            slot = i * slots + j
            assert sizes[slot] == len(block), (i, j)
            if with_bytes:
                got = host[slot * slot_bytes:slot * slot_bytes + len(block)].tobytes()
                assert got == block, (i, j)
                assert model.decode(got) == piece
            want_counts[0] += 1
            want_counts[1] += len(piece)
            want_counts[2] += min(len(block), len(piece))
            want_counts[3] += len(block) >= len(piece)
    return tuple(want_counts)


KINDS = ["zero", "random", "acgt", "text", "blockvar"]


@pytest.mark.parametrize("shift", [12, 13, 14, 15, 16, 17, 18, 19, 20])
def test_kernel_matches_the_model(cuda_device, shift):
    """per chunk size: one descriptor per kind of data, ragged last chunks, odd device addresses"""
    chunk = 1 << shift
    rng = np.random.default_rng(shift)
    lens = [2 * chunk, chunk + int(rng.integers(1, chunk)), int(rng.integers(1, 40)), chunk - 3,
            3 * chunk + 13]
    datas = [make_data(kind, n, shift * 10 + i) for i, (kind, n) in enumerate(zip(KINDS, lens))]
    slots = 4
    buf = torch.zeros(sum(n + 64 for n in lens), dtype=torch.uint8, device="cuda")
    blocks, pos = [], 0
    for i, data in enumerate(datas):
        off = pos + (i * 7) % 5  # (odd addresses)
        buf[off:off + len(data)] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
        blocks.append((buf, off, len(data), (i + 1) << 20))
        pos += len(data) + 64
    counters = torch.zeros(4, dtype=torch.int64, device="cuda")
    keep = _launch(blocks, shift, slots, counters)
    torch.cuda.synchronize()
    want = _check_against_model(datas, shift, blocks, slots, keep[1], keep[2])
    assert tuple(counters.cpu().tolist()) == want
    # the size-only path gives the same counts
    counters.zero_()
    keep2 = _launch(blocks, shift, slots, counters, with_bytes=False)
    torch.cuda.synchronize()
    assert torch.equal(keep2[1], keep[1])
    assert tuple(counters.cpu().tolist()) == want


def test_many_descriptors_and_long_matches(cuda_device):
    """64 descriptors of 1 MiB chunks mixing long zero runs, repeats further back than 64 KiB and
    random data"""
    shift, n = 20, 64
    rng = np.random.default_rng(9)
    datas = []
    for i in range(n):
        r = rng.integers(0, 256, 80 * KiB, dtype=np.uint8).tobytes()
        datas.append((r + bytes(int(rng.integers(0, 300 * KiB))) + r + r[:1000])[:MiB])
    buf = torch.frombuffer(bytearray(b"".join(datas)), dtype=torch.uint8).cuda()
    offs = np.cumsum([0] + [len(d) for d in datas])
    blocks = [(buf, int(offs[i]), len(datas[i]), 0) for i in range(n)]
    counters = torch.zeros(4, dtype=torch.int64, device="cuda")
    keep = _launch(blocks, shift, 1, counters)
    torch.cuda.synchronize()
    assert tuple(counters.cpu().tolist()) == _check_against_model(datas, shift, blocks, 1,
                                                                   keep[1], keep[2])


def test_block_past_4gib(cuda_device):
    """one descriptor of 4 GiB + 192 KiB, chunks of 64 KiB: the chunks past 4 GiB are right"""
    shift, length = 16, 4 * GiB + 192 * KiB
    big = torch.zeros(length, dtype=torch.uint8, device="cuda")
    tail = make_data("text", 192 * KiB + 64 * KiB, 3)
    big[4 * GiB - 64 * KiB:] = torch.frombuffer(bytearray(tail), dtype=torch.uint8).cuda()
    slots = length >> shift
    counters = torch.zeros(4, dtype=torch.int64, device="cuda")
    keep = _launch([(big, 0, length, 0)], shift, slots, counters, with_bytes=False)
    torch.cuda.synchronize()
    sizes = keep[1].cpu().numpy()
    zero_size = model.size(bytes(64 * KiB))
    assert (sizes[:slots - 4] == zero_size).all()
    for j in range(4):
        assert sizes[slots - 4 + j] == model.size(tail[j * 64 * KiB:(j + 1) * 64 * KiB])
    del big


def test_two_streams_into_one_block(cuda_device):
    shift = 16
    datas = [make_data(kind, 512 * KiB + 100, 20 + i) for i, kind in enumerate(KINDS)]
    bufs = [torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda() for d in datas]
    counters = torch.zeros(4, dtype=torch.int64, device="cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    keep = [_launch([(b, 0, len(d), 0) for b, d in zip(bufs[:3], datas[:3])], shift, 9, counters,
                    s1, False),
            _launch([(b, 0, len(d), 0) for b, d in zip(bufs[3:], datas[3:])], shift, 9, counters,
                    s2, False)]
    torch.cuda.synchronize()
    assert tuple(counters.cpu().tolist()) == model.counts(datas, 64 * KiB)
    del keep


# ---- the setter --------------------------------------------------------------------------

@pytest.mark.parametrize("extra,message", [
    (dict(compress_chunk=2 * KiB), "The compress chunk shift (11) is not in [12, 20]."),
    (dict(compress_chunk=2 * MiB), "The compress chunk shift (21) is not in [12, 20]."),
    (dict(compress_chunk=3 * KiB), "The compress chunk shift (4294967295) is not in [12, 20]."),
    (dict(compress_chunk=512 * KiB), "The block size (262144) is not a multiple of the compress "
                                     "chunk size (--compressstats) (524288)."),
    (dict(compress_chunk=64 * KiB, use_random_offsets=True, use_random_unaligned=True),
     "Compress stats (--compressstats) cannot be used together with unaligned random offsets "
     "(--norandalign)."),
    (dict(compress_chunk=64 * KiB, rwmix_read_percent=50),
     "Compress stats (--compressstats) cannot be used together with rwmix (a phase in both "
     "directions)."),
    (dict(compress_chunk=64 * KiB, num_threads=2, num_rwmix_read_threads=1),
     "Compress stats (--compressstats) cannot be used together with rwmix (a phase in both "
     "directions)."),
])
def test_setter_rejections(tmp_path, cuda_device, extra, message):
    cfg = WorkerConfig(paths=[str(tmp_path / "f")], block_size=256 * KiB, file_size=4 * MiB,
                       **extra)
    with pytest.raises(WorkerError) as excinfo:
        WorkerManager(cfg)
    assert str(excinfo.value) == message


def test_setter_through_ctypes(tmp_path, cuda_device):
    lib = _native.load()
    cfg = WorkerConfig(paths=[str(tmp_path / "f")], block_size=256 * KiB, file_size=4 * MiB)
    with WorkerManager(cfg) as mgr:
        out = [ctypes.c_uint64(7) for _ in range(4)]
        assert lib.elb_mgr_compress_stats(mgr._h, *[ctypes.byref(v) for v in out]) == -1
        assert _native.last_error() == ("elb_mgr_compress_stats: compress stats are off "
                                        "(elb_mgr_set_compress_stats)")
        for shift in (1, 11, 21, 64):
            assert lib.elb_mgr_set_compress_stats(mgr._h, shift) == -1
            assert _native.last_error() == ("The compress chunk shift (%d) is not in [12, 20]."
                                            % shift)
        assert lib.elb_mgr_set_compress_stats(mgr._h, 19) == -1
        assert lib.elb_mgr_set_compress_stats(mgr._h, 18) == 0
        assert mgr.compress_stats() == (0, 0, 0, 0)  # (no phase yet)
        assert lib.elb_mgr_set_compress_stats(mgr._h, 0) == 0
        with pytest.raises(WorkerError):
            mgr.compress_stats()


# ---- the worker ----------------------------------------------------------------------------

@pytest.fixture()
def workdir(cuda_device):
    path = make_workdir()
    yield path
    shutil.rmtree(path, ignore_errors=True)


def expected_counts(paths, chunk):
    datas = []
    for path in paths:
        with open(path, "rb") as f:
            datas.append(f.read())
    return model.counts(datas, chunk)


def run_phases(cfg_args, phases=(BenchPhase.CREATEFILES, BenchPhase.READFILES)):
    out = []
    with WorkerManager(WorkerConfig(**cfg_args)) as mgr:
        for phase in phases:
            res = mgr.run_phase(phase)
            out.append((mgr.compress_stats(), res["num_kernel_launches"]))
    return out


@pytest.mark.parametrize("content", [dict(block_variance_percent=0),
                                     dict(block_variance_percent=50),
                                     dict(block_variance_percent=100),
                                     dict(integrity_check_salt=7,
                                          integrity_check_kind=kernels.VERIFY_RANDOM,
                                          block_variance_percent=50)],
                         ids=["var0", "var50", "var100", "verifyrand50"])
@pytest.mark.parametrize("variant", [
    dict(block_size=64 * KiB), dict(block_size=256 * KiB, num_threads=4),
    dict(block_size=64 * KiB, io_engine=IOEngine.AIO, io_depth=8),
    dict(block_size=64 * KiB, staging_engine=1), dict(block_size=64 * KiB, staging_engine=2),
    dict(block_size=64 * KiB, use_direct_io=True), dict(block_size=64 * KiB, use_cufile=True),
], ids=["64K", "threads4", "aio8", "kernel", "copyengine", "direct", "cufile"])
def test_counts_match_the_files(variant, content, cuda_device):
    whole = variant.get("use_direct_io") or variant.get("use_cufile")
    workdir = make_workdir(direct=bool(whole))
    try:
        paths = [os.path.join(workdir, "f%d" % i) for i in range(2)]
        size = 2 * MiB + (0 if whole else 20 * KiB)  # (a short last chunk unless whole blocks)
        out = run_phases(dict(paths=paths, file_size=size, compress_chunk=16 * KiB, **content,
                              **variant))
        want = expected_counts(paths, 16 * KiB)
        assert out[0][0] == want and out[1][0] == want
    finally:
        shutil.rmtree(workdir, ignore_errors=True)


def test_dir_mode(workdir):
    args = dict(paths=[workdir], path_type=PathType.DIR, num_dirs=2, num_files=3,
                num_threads=2, block_size=128 * KiB, file_size=512 * KiB + 4 * KiB,
                block_variance_percent=50, compress_chunk=4 * KiB)
    out = run_phases(args, phases=(BenchPhase.CREATEDIRS, BenchPhase.CREATEFILES,
                                   BenchPhase.READFILES))[1:]
    files = [os.path.join(root, f) for root, _, names in os.walk(workdir) for f in names]
    assert len(files) == 12
    want = expected_counts(sorted(files), 4 * KiB)
    assert out[0][0] == want and out[1][0] == want


def test_custom_tree_mode(workdir):
    tree_path = os.path.join(workdir, "tree.txt")
    bench_dir = os.path.join(workdir, "bench")
    os.mkdir(bench_dir)
    with open(tree_path, "w") as f:
        f.write(TREE_TEXT)
    _, files = tree_model.parse_tree(TREE_TEXT)
    out = run_phases(dict(paths=[bench_dir], path_type=PathType.DIR, num_threads=3,
                          block_size=64 * KiB, block_variance_percent=40,
                          tree_file_path=tree_path, compress_chunk=16 * KiB),
                     phases=(BenchPhase.CREATEDIRS, BenchPhase.CREATEFILES,
                             BenchPhase.READFILES))[1:]
    want = expected_counts([os.path.join(bench_dir, p) for p, _ in files], 16 * KiB)
    assert out[0][0] == want and out[1][0] == want


def test_random_read_of_uniform_data(workdir):
    """every 64 KiB chunk of the file is the same text, so a --rand read of N chunks stores N
    times the size of one"""
    path = os.path.join(workdir, "f")
    piece = make_data("text", 64 * KiB, 1)
    with open(path, "wb") as f:
        f.write(piece * 64)
    out = run_phases(dict(paths=[path], file_size=4 * MiB, block_size=256 * KiB,
                          use_random_offsets=True, random_amount=24 * MiB, compress_chunk=64 * KiB),
                     phases=(BenchPhase.READFILES,))
    n = 24 * MiB // (64 * KiB)
    s = model.size(piece)
    assert out[0][0] == (n, 24 * MiB, n * s, 0)


def test_last_data_set_thread_takes_the_remainder(workdir):
    """one 30 MiB + 5 KiB file of 1 MiB blocks over 16 data set threads, of which this process
    runs the last (--rankoffset 15): its 16 blocks and the short tail"""
    path = os.path.join(workdir, "f")
    size = 30 * MiB + 5 * KiB
    with open(path, "wb") as f:
        f.write(make_data("blockvar", size, 4))
    out = run_phases(dict(paths=[path], file_size=size, block_size=MiB, num_threads=1,
                          rank_offset=15, num_dataset_threads=16, compress_chunk=4 * KiB),
                     phases=(BenchPhase.READFILES,))
    with open(path, "rb") as f:
        f.seek(15 * MiB)
        tail = f.read()
    assert out[0][0] == model.counts([tail], 4 * KiB)


def test_two_gpus_add_up(workdir):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    paths = [os.path.join(workdir, "f%d" % i) for i in range(4)]
    args = dict(paths=paths, file_size=2 * MiB, block_size=256 * KiB, num_threads=4,
                block_variance_percent=50, compress_chunk=16 * KiB)
    one = run_phases(dict(args, gpu_ids=(0,)))
    two = run_phases(dict(args, gpu_ids=(0, 1)), phases=(BenchPhase.READFILES,))
    assert two[0][0] == one[1][0] == expected_counts(paths, 16 * KiB)


def test_launches_and_copies(workdir):
    """without --compressstats a phase launches and copies what it did before: one fill / verify
    launch per batch, the data once each way; with it, one LZ4 launch per batch more and no copy.
    A chunk size set between phases takes effect in the next one."""
    path = os.path.join(workdir, "f")
    size, block, batch_blocks = 8 * MiB, MiB, 2
    num_batches = size // block // batch_blocks
    counters = {}
    for chunk in (0, 64 * KiB):
        cfg = WorkerConfig(paths=[path], file_size=size, block_size=block,
                           pipeline_batch_blocks=batch_blocks, integrity_check_salt=5,
                           staging_engine=2, compress_chunk=chunk)
        with WorkerManager(cfg) as mgr:
            for phase in (BenchPhase.CREATEFILES, BenchPhase.READFILES):
                r = mgr.run_phase(phase)
                counters[chunk, phase] = (r["num_kernel_launches"], r["h2d_bytes"],
                                          r["d2h_bytes"])
            if not chunk:
                with pytest.raises(WorkerError, match="compress stats are off"):
                    mgr.compress_stats()
                assert _native.load().elb_mgr_set_compress_stats(mgr._h, 12) == 0
                r = mgr.run_phase(BenchPhase.READFILES)
                assert r["num_kernel_launches"] == 2 * num_batches
                assert mgr.compress_stats() == expected_counts([path], 4 * KiB)
    assert counters[0, BenchPhase.CREATEFILES] == (num_batches, 0, size)
    assert counters[0, BenchPhase.READFILES] == (num_batches, size, 0)
    assert counters[64 * KiB, BenchPhase.CREATEFILES] == (2 * num_batches, 0, size)
    assert counters[64 * KiB, BenchPhase.READFILES] == (2 * num_batches, size, 0)


def test_cli_prints_the_line(workdir):
    path = os.path.join(workdir, "f")
    res = run_cli("-w", "-r", "-b", "1m", "-s", "8m", "--gpuids", "0", "--blockvarpct", "50",
                  "--compressstats", "64k", path)
    assert res.returncode == 0, res.stderr
    lines = [line for line in res.stdout.splitlines() if line.startswith("Compress: ")]
    assert len(lines) == 2 and lines[0] == lines[1]
    n, b, s, u = expected_counts([path], 64 * KiB)
    assert lines[0] == kernels.compress_line(64 * KiB, n, b, s, u)
    assert n == 128 and s < b
