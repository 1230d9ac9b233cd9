"""GPU tests of --reducestats: the insert marks one slot per distinct key across two streams, the
masked LZ4 launch writes the payloads of tests/reduce_model.py for each distinct chunk (chunk sizes
4K, 64K and 1M, ragged chunks, odd addresses, a block past 4 GiB) and none for the other slots, a
merge carries payloads and adds nothing the second time, the sum kernel, the overflow flag and the
setter; then the worker's (N, D, B, U, S) against the model applied to the files on disk
(--dedupepct, --blockvarpct, zero files, block sizes, threads, AIO, staging engines, --direct,
mock cuFile, dir mode, custom tree mode, two GPUs), next to --dedupestats and --compressstats, the
launches and copies with and without the option, and the console line of the command line."""
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
from tests import compress_model  # noqa: E402
from tests import reduce_model as model  # noqa: E402
from tests import tree_model  # noqa: E402
from tests.test_compress_stats import make_data  # noqa: E402
from tests.test_custom_tree_gpu import TREE_TEXT  # noqa: E402
from tests.test_checksums_gpu import make_workdir, run_cli  # noqa: E402

pytestmark = pytest.mark.gpu

KiB, MiB, GiB = 1 << 10, 1 << 20, 1 << 30
NOT_NEW = kernels.REDUCE_NOT_NEW


class Table:
    """a reduce table on the current GPU: keys, payloads and counters"""

    def __init__(self, entries):
        self.entries = entries
        self.mem = torch.zeros(entries * (16 + kernels.REDUCE_PAYLOAD_BYTES), dtype=torch.uint8,
                               device="cuda")
        self.keys_ptr = self.mem.data_ptr()
        self.payloads_ptr = self.keys_ptr + 16 * entries
        self.counters = torch.zeros(kernels.REDUCE_COUNTERS_BYTES, dtype=torch.uint8,
                                    device="cuda")

    def keys(self):
        return self.mem[:16 * self.entries].cpu().numpy().reshape(-1, 16)

    def payloads(self):
        return self.mem[16 * self.entries:].cpu().numpy().view("<u4").reshape(-1, 2)

    def read_counters(self):
        return kernels.reduce_counters(self.counters.cpu().numpy().tobytes())

    def stored(self):
        """{key: (length, stored)} of the entries with a key"""
        keys, payloads = self.keys(), self.payloads()
        used = np.nonzero(keys.any(axis=1))[0]
        return {keys[e].tobytes(): tuple(int(x) for x in payloads[e]) for e in used}

    def sum(self, stream=0):
        kernels.reduce_sum(self.keys_ptr, self.payloads_ptr, self.entries,
                           self.counters.data_ptr(), stream)


def _pinned_descs(blocks):
    raw = kernels.pack_block_descs([(t.data_ptr() + o, n, f, 0) for t, o, n, f in blocks])
    return torch.frombuffer(bytearray(raw), dtype=torch.uint8).pin_memory()


def _launch(blocks, shift, slots, table, stream=None):
    """blocks: [(device tensor, byte offset in it, length, file offset)]: digests, insert and
    masked LZ4 on one stream -> (descs, digests, marks) tensors"""
    descs = _pinned_descs(blocks)
    digests = torch.zeros(len(blocks) * slots * 32, dtype=torch.uint8, device="cuda")
    marks = torch.full((len(blocks) * slots,), -1, dtype=torch.int64, device="cuda")
    s = stream or torch.cuda.current_stream()
    with torch.cuda.stream(s):
        kernels.blake3_chunks(descs.data_ptr(), 0, len(blocks), shift, slots, digests.data_ptr(),
                              stream=s.cuda_stream)
        kernels.reduce_insert(descs.data_ptr(), len(blocks), shift, slots, digests.data_ptr(),
                              table.keys_ptr, table.entries, table.counters.data_ptr(),
                              marks.data_ptr(), s.cuda_stream)
        kernels.reduce_lz4(descs.data_ptr(), len(blocks), shift, slots, marks.data_ptr(),
                           table.payloads_ptr, s.cuda_stream)
    return descs, digests, marks


def _place(datas, odd=True):
    """the datas in one device buffer at odd offsets -> blocks with chunk-aligned file offsets"""
    buf = torch.zeros(sum(len(d) + 64 for d in datas), dtype=torch.uint8, device="cuda")
    blocks, pos = [], 0
    for i, data in enumerate(datas):
        off = pos + ((i * 7) % 5 if odd else 0)
        if data:
            buf[off:off + len(data)] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
        blocks.append((buf, off, len(data), i << 30))
        pos += len(data) + 64
    return buf, blocks


def _model_stored(datas, chunk):
    """{key: (length, stored)} of the distinct chunks of datas"""
    out = {}
    for data in datas:
        for j, key in enumerate(model.chunk_keys(data, chunk)):
            piece = data[j * chunk:(j + 1) * chunk]
            out.setdefault(key, (len(piece), min(compress_model.size(piece), len(piece))))
    return out


def _mixed_datas(shift, seed):
    """descriptors of several kinds with repeated chunks and ragged last chunks"""
    chunk = 1 << shift
    rng = np.random.default_rng(seed)
    text = make_data("text", chunk, seed)
    rand = make_data("random", chunk, seed + 1)
    tail = make_data("acgt", int(rng.integers(1, chunk)), seed + 2)
    return [text + rand + text + tail, bytes(2 * chunk) + text, rand + bytes(chunk - 3),
            tail, make_data("blockvar", 3 * chunk + 13, seed + 3) + b"", text + rand + tail]


# ---- the kernels ---------------------------------------------------------------------------

@pytest.mark.parametrize("shift", [12, 16, 20])
def test_payloads_match_the_model(cuda_device, shift):
    chunk = 1 << shift
    datas = _mixed_datas(shift, shift)
    slots = max((len(d) + chunk - 1) // chunk for d in datas)
    buf, blocks = _place(datas)
    table = Table(1024)
    keep = _launch(blocks, shift, slots, table)
    table.sum()
    torch.cuda.synchronize()
    want = _model_stored(datas, chunk)
    assert table.stored() == want
    n, d, b, u, s = model.counts(datas, chunk)
    assert table.read_counters() == (n, b, d, u, s, 0)
    # one marked slot per distinct key, and its entry holds the key
    marks = keep[2].cpu().numpy().view(np.uint64)
    marked = marks[marks != NOT_NEW]
    assert len(marked) == d and len(set(marked.tolist())) == d
    keys = table.keys()
    assert set(keys[int(e)].tobytes() for e in marked) == set(want)
    # entries without a key have no payload
    payloads = table.payloads()
    assert not payloads[~keys.any(axis=1)].any()
    del buf


def test_two_streams_mark_one_slot_per_key(cuda_device):
    """the same chunks inserted from two streams at once: each distinct key is marked once, its
    payload written once"""
    shift, chunk = 12, 4 * KiB
    pool = [make_data("text", chunk, i) for i in range(300)] + [bytes(chunk)]
    rng = np.random.default_rng(5)
    datas = [b"".join(pool[k] for k in rng.integers(0, len(pool), 64)) for _ in range(32)]
    buf, blocks = _place(datas, odd=False)
    table = Table(4096)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    keep = [_launch(blocks, shift, 64, table, s1), _launch(blocks, shift, 64, table, s2)]
    torch.cuda.synchronize()
    table.sum()
    torch.cuda.synchronize()
    marks = np.concatenate([k[2].cpu().numpy().view(np.uint64) for k in keep])
    marked = marks[marks != NOT_NEW]
    want = _model_stored(datas, chunk)
    assert len(marked) == len(want) == len(set(marked.tolist()))
    assert table.stored() == want
    n, d, b, u, s = model.counts(datas, chunk)
    assert table.read_counters() == (2 * n, 2 * b, d, u, s, 0)
    del buf


def test_block_past_4gib(cuda_device):
    """one descriptor of 4 GiB + 192 KiB, chunks of 64 KiB: zeros, then text from 4 GiB - 64 KiB"""
    shift, length = 16, 4 * GiB + 192 * KiB
    big = torch.zeros(length, dtype=torch.uint8, device="cuda")
    tail = make_data("text", 256 * KiB, 3)
    big[4 * GiB - 64 * KiB:] = torch.frombuffer(bytearray(tail), dtype=torch.uint8).cuda()
    slots = length >> shift
    table = Table(1024)
    keep = _launch([(big, 0, length, 0)], shift, slots, table)
    table.sum()
    torch.cuda.synchronize()
    pieces = [tail[j * 64 * KiB:(j + 1) * 64 * KiB] for j in range(4)]
    want = _model_stored([bytes(64 * KiB)] + pieces, 64 * KiB)
    assert table.stored() == want
    n, b = slots, length
    u = sum(v[0] for v in want.values())
    s = sum(v[1] for v in want.values())
    assert table.read_counters() == (n, b, len(want), u, s, 0)
    del keep, big


def test_merge_carries_payloads(cuda_device):
    shift, chunk = 14, 16 * KiB
    shared_data = make_data("text", 8 * chunk, 1)
    a_datas = [shared_data + make_data("blockvar", 4 * chunk, 2)]
    b_datas = [make_data("acgt", 5 * chunk + 77, 3) + b"", shared_data]
    table_a, table_b = Table(1024), Table(256)
    buf_a, blocks_a = _place(a_datas)
    buf_b, blocks_b = _place(b_datas)
    keep = [_launch(blocks_a, shift, 16, table_a), _launch(blocks_b, shift, 16, table_b)]
    torch.cuda.synchronize()
    kernels.reduce_merge(table_b.keys_ptr, table_b.payloads_ptr, table_b.entries,
                         table_a.keys_ptr, table_a.payloads_ptr, table_a.entries,
                         table_a.counters.data_ptr())
    torch.cuda.synchronize()
    merged = table_a.mem.clone()
    assert table_a.stored() == _model_stored(a_datas + b_datas, chunk)
    # a second merge adds nothing
    kernels.reduce_merge(table_b.keys_ptr, table_b.payloads_ptr, table_b.entries,
                         table_a.keys_ptr, table_a.payloads_ptr, table_a.entries,
                         table_a.counters.data_ptr())
    table_a.sum()
    torch.cuda.synchronize()
    assert torch.equal(table_a.mem, merged)
    _, d, _, u, s = model.counts(a_datas + b_datas, chunk)
    counters = table_a.read_counters()
    assert counters[2:] == (d, u, s, 0)
    del keep, buf_a, buf_b


def test_sum_kernel(cuda_device):
    """hand-written entries: the sum counts the entries with a key and adds their payloads"""
    entries = 1 << 16
    table = Table(entries)
    rng = np.random.default_rng(7)
    used = rng.choice(entries, 5000, replace=False)
    keys = np.zeros((entries, 16), dtype=np.uint8)
    keys[used] = rng.integers(0, 256, (len(used), 16), dtype=np.uint8)
    keys[used, 0] |= 1
    payloads = np.zeros((entries, 2), dtype="<u4")
    payloads[used, 0] = rng.integers(1, MiB + 1, len(used))
    payloads[used, 1] = payloads[used, 0] // 3
    unused = np.setdiff1d(np.arange(entries), used)[:100]
    payloads[unused] = 5  # (only entries with a key count)
    table.mem.copy_(torch.from_numpy(np.concatenate([keys.reshape(-1),
                                                     payloads.view(np.uint8).reshape(-1)])))
    table.sum()
    torch.cuda.synchronize()
    assert table.read_counters() == (0, 0, 5000, int(payloads[used, 0].sum()),
                                     int(payloads[used, 1].sum()), 0)


def test_overflow_flag(cuda_device):
    """2048 distinct chunks into 1024 entries: the probe bound is hit and the flag set"""
    shift = 12
    data = make_data("random", 2048 * 4 * KiB, 8)
    buf, blocks = _place([data], odd=False)
    table = Table(1024)
    keep = _launch(blocks, shift, 2048, table)
    torch.cuda.synchronize()
    counters = table.read_counters()
    assert counters[0] == 2048 and counters[5] == 1
    marks = keep[2].cpu().numpy().view(np.uint64)
    assert (marks != NOT_NEW).sum() == 1024
    del buf


# ---- the setter ----------------------------------------------------------------------------

@pytest.mark.parametrize("extra,message", [
    (dict(reduce_chunk=2 * KiB), "The reduce chunk shift (11) is not in [12, 20]."),
    (dict(reduce_chunk=2 * MiB), "The reduce chunk shift (21) is not in [12, 20]."),
    (dict(reduce_chunk=3 * KiB), "The reduce chunk shift (4294967295) is not in [12, 20]."),
    (dict(reduce_chunk=512 * KiB), "The block size (262144) is not a multiple of the reduce "
                                   "chunk size (--reducestats) (524288)."),
    (dict(reduce_chunk=64 * KiB, use_random_offsets=True),
     "Reduce stats (--reducestats) cannot be used together with random offsets (--rand)."),
    (dict(reduce_chunk=64 * KiB, do_infinite_io_loop=True),
     "Reduce stats (--reducestats) cannot be used together with an infinite I/O loop "
     "(--infloop)."),
    (dict(reduce_chunk=64 * KiB, rwmix_read_percent=50),
     "Reduce stats (--reducestats) cannot be used together with rwmix (a phase in both "
     "directions)."),
    (dict(reduce_chunk=64 * KiB, num_threads=2, num_rwmix_read_threads=1),
     "Reduce stats (--reducestats) cannot be used together with rwmix (a phase in both "
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
        out = [ctypes.c_uint64(7) for _ in range(5)]
        assert lib.elb_mgr_reduce_stats(mgr._h, *[ctypes.byref(v) for v in out]) == -1
        assert _native.last_error() == ("elb_mgr_reduce_stats: reduce stats are off "
                                        "(elb_mgr_set_reduce_stats)")
        for shift in (1, 11, 21, 64):
            assert lib.elb_mgr_set_reduce_stats(mgr._h, shift) == -1
            assert _native.last_error() == ("The reduce chunk shift (%d) is not in [12, 20]."
                                            % shift)
        assert lib.elb_mgr_set_reduce_stats(mgr._h, 19) == -1
        assert lib.elb_mgr_set_reduce_stats(mgr._h, 18) == 0
        assert mgr.reduce_stats() == (0, 0, 0, 0, 0)  # (no phase yet)
        assert lib.elb_mgr_set_reduce_stats(mgr._h, 0) == 0
        with pytest.raises(WorkerError):
            mgr.reduce_stats()


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


def run_phases(cfg_args, phases=(BenchPhase.CREATEFILES, BenchPhase.READFILES), also=()):
    out = []
    with WorkerManager(WorkerConfig(**cfg_args)) as mgr:
        for phase in phases:
            res = mgr.run_phase(phase)
            out.append((mgr.reduce_stats(), res["num_kernel_launches"],
                        tuple(getattr(mgr, name)() for name in also)))
    return out


GRAIN = 16 * KiB


@pytest.mark.parametrize("dedupe_pct", [0, 50, 100])
def test_dedupe_percent(workdir, dedupe_pct):
    paths = [os.path.join(workdir, "f%d" % i) for i in range(2)]
    content = dict(integrity_check_salt=11, integrity_check_kind=kernels.VERIFY_RANDOM,
                   verify_random_grain=GRAIN, dedupe_percent=dedupe_pct,
                   block_variance_percent=50)
    out = run_phases(dict(paths=paths, file_size=2 * MiB, block_size=256 * KiB, num_threads=2,
                          reduce_chunk=GRAIN, **content))
    want = expected_counts(paths, GRAIN)
    assert out[0][0] == want and out[1][0] == want
    if dedupe_pct == 100:
        assert want[1] < want[0]


CONTENTS = [dict(block_variance_percent=0), dict(block_variance_percent=50)]


@pytest.mark.parametrize("content", CONTENTS, ids=["var0", "var50"])
@pytest.mark.parametrize("variant", [
    dict(block_size=16 * KiB), dict(block_size=64 * KiB, num_threads=8),
    dict(block_size=64 * KiB, io_engine=IOEngine.AIO, io_depth=8),
    dict(block_size=64 * KiB, staging_engine=1), dict(block_size=64 * KiB, staging_engine=2),
    dict(block_size=64 * KiB, use_direct_io=True), dict(block_size=64 * KiB, use_cufile=True),
], ids=["K", "threads8", "aio8", "kernel", "copyengine", "direct", "cufile"])
def test_counts_match_the_files(variant, content, cuda_device):
    whole = variant.get("use_direct_io") or variant.get("use_cufile")
    workdir = make_workdir(direct=bool(whole))
    try:
        paths = [os.path.join(workdir, "f%d" % i) for i in range(2)]
        size = MiB + (0 if whole else 20 * KiB)  # (a short last chunk unless whole blocks)
        out = run_phases(dict(paths=paths, file_size=size, reduce_chunk=16 * KiB, **content,
                              **variant))
        want = expected_counts(paths, 16 * KiB)
        assert out[0][0] == want and out[1][0] == want
    finally:
        shutil.rmtree(workdir, ignore_errors=True)


def test_zero_files_with_a_short_last_chunk(workdir):
    paths = [os.path.join(workdir, "f%d" % i) for i in range(3)]
    for path in paths:
        with open(path, "wb") as f:
            f.write(bytes(MiB + 5 * KiB))
    out = run_phases(dict(paths=paths, file_size=MiB + 5 * KiB, block_size=64 * KiB,
                          num_threads=2, reduce_chunk=64 * KiB), phases=(BenchPhase.READFILES,))
    zero, short = compress_model.size(bytes(64 * KiB)), compress_model.size(bytes(5 * KiB))
    assert out[0][0] == (3 * 17, 2, 3 * (MiB + 5 * KiB), 69 * KiB, zero + short)


def test_dir_mode(workdir):
    args = dict(paths=[workdir], path_type=PathType.DIR, num_dirs=2, num_files=3,
                num_threads=2, block_size=128 * KiB, file_size=256 * KiB + 4 * KiB,
                block_variance_percent=50, reduce_chunk=4 * KiB)
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
                          tree_file_path=tree_path, reduce_chunk=16 * KiB),
                     phases=(BenchPhase.CREATEDIRS, BenchPhase.CREATEFILES,
                             BenchPhase.READFILES))[1:]
    want = expected_counts([os.path.join(bench_dir, p) for p, _ in files], 16 * KiB)
    assert out[0][0] == want and out[1][0] == want


def test_two_gpus_give_the_result_of_one(workdir):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    paths = [os.path.join(workdir, "f%d" % i) for i in range(4)]
    args = dict(paths=paths, file_size=MiB, block_size=256 * KiB, num_threads=4,
                integrity_check_salt=3, integrity_check_kind=kernels.VERIFY_RANDOM,
                verify_random_grain=GRAIN, dedupe_percent=50, reduce_chunk=GRAIN)
    one = run_phases(dict(args, gpu_ids=(0,)))
    two = run_phases(dict(args, gpu_ids=(0, 1)), phases=(BenchPhase.READFILES,))
    assert two[0][0] == one[1][0] == one[0][0] == expected_counts(paths, GRAIN)


@pytest.mark.parametrize("dedupe_chunk", [GRAIN, 4 * KiB])
def test_next_to_dedupe_stats(workdir, dedupe_chunk):
    """N and D agree with --dedupestats at the same chunk size, whose BLAKE3 launch is shared"""
    paths = [os.path.join(workdir, "f%d" % i) for i in range(2)]
    out = run_phases(dict(paths=paths, file_size=MiB, block_size=256 * KiB,
                          integrity_check_salt=9, integrity_check_kind=kernels.VERIFY_RANDOM,
                          verify_random_grain=GRAIN, dedupe_percent=50, reduce_chunk=GRAIN,
                          dedupe_chunk=dedupe_chunk), also=("dedupe_stats",))
    want = expected_counts(paths, GRAIN)
    for stats, _, (dedupe,) in out:
        assert stats == want
        if dedupe_chunk == GRAIN:
            assert dedupe[:2] == stats[:2]


def test_next_to_compress_stats(workdir):
    """on data without duplicates S is what --compressstats stores"""
    paths = [os.path.join(workdir, "f%d" % i) for i in range(2)]
    out = run_phases(dict(paths=paths, file_size=MiB, block_size=256 * KiB,
                          integrity_check_salt=9, integrity_check_kind=kernels.VERIFY_RANDOM,
                          verify_random_grain=4 * KiB, block_variance_percent=50,
                          reduce_chunk=64 * KiB, compress_chunk=64 * KiB),
                     also=("compress_stats",))
    for stats, _, (compress,) in out:
        n, d, b, u, s = stats
        assert d == n and u == b
        assert (compress[0], compress[1], compress[2]) == (n, b, s)


def test_next_to_blake3_checksums(workdir):
    """the BLAKE3 launch of --checksums at the same chunk size is shared"""
    paths = [os.path.join(workdir, "f%d" % i) for i in range(2)]
    out = run_phases(dict(paths=paths, file_size=MiB, block_size=256 * KiB,
                          block_variance_percent=50, checksums=True, checksum_algo="blake3",
                          checksum_chunk_shift=14, reduce_chunk=16 * KiB))
    want = expected_counts(paths, 16 * KiB)
    assert out[0][0] == want and out[1][0] == want


def test_launches_and_copies(workdir):
    """without --reducestats a phase launches and copies what it did before: one fill / verify
    launch per batch, the data once each way; with it, three launches per batch more (BLAKE3,
    insert, LZ4) and no copy"""
    path = os.path.join(workdir, "f")
    size, block, batch_blocks = 8 * MiB, MiB, 2
    num_batches = size // block // batch_blocks
    counters = {}
    for chunk in (0, 64 * KiB):
        cfg = WorkerConfig(paths=[path], file_size=size, block_size=block,
                           pipeline_batch_blocks=batch_blocks, integrity_check_salt=5,
                           staging_engine=2, reduce_chunk=chunk)
        with WorkerManager(cfg) as mgr:
            for phase in (BenchPhase.CREATEFILES, BenchPhase.READFILES):
                r = mgr.run_phase(phase)
                counters[chunk, phase] = (r["num_kernel_launches"], r["h2d_bytes"],
                                          r["d2h_bytes"])
            if not chunk:
                with pytest.raises(WorkerError, match="reduce stats are off"):
                    mgr.reduce_stats()
    assert counters[0, BenchPhase.CREATEFILES] == (num_batches, 0, size)
    assert counters[0, BenchPhase.READFILES] == (num_batches, size, 0)
    assert counters[64 * KiB, BenchPhase.CREATEFILES] == (4 * num_batches, 0, size)
    assert counters[64 * KiB, BenchPhase.READFILES] == (4 * num_batches, size, 0)


def test_cli_prints_the_line(workdir):
    path = os.path.join(workdir, "f")
    res = run_cli("-w", "-r", "-t", "2", "-b", "1m", "-s", "8m", "--gpuids", "0",
                  "--verifyrand", "7", "--verifyrandgrain", "64k", "--dedupepct", "50",
                  "--blockvarpct", "50", "--reducestats", "64k", path)
    assert res.returncode == 0, res.stderr
    lines = [line for line in res.stdout.splitlines() if line.startswith("Reduce: ")]
    assert len(lines) == 2 and lines[0] == lines[1]
    n, d, b, u, s = expected_counts([path], 64 * KiB)
    assert lines[0] == model.line(64 * KiB, n, d, b, u, s)
    assert n == 128 and s < u
