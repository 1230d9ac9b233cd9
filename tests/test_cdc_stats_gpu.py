"""GPU tests of --cdcstats: the cut kernel's chunks equal tests/cdc_model.py exactly (random, zero
and --blockvarpct data; AVG 4K, 16K and 256K; ragged descriptors; odd addresses; many descriptors
per launch; a block past 4 GiB), every digest of the hash-insert launch is blake3 of its chunk and
the table holds the model's distinct chunks (also from two streams, and merged from two tables),
a too-small table sets the overflow flag; then the worker's (N, D, B, U) against the model applied
to the files on disk across block sizes, threads, AIO, staging engines, --direct, mock cuFile, dir
mode, custom tree mode and --dedupepct data, the shifted copy that fixed-offset dedupe cannot see,
the other stats options next to it, launches and copies, and the console line."""
import os
import shutil

import blake3
import numpy as np
import pytest
import torch

from tests import test_checksums_gpu as base  # noqa: F401  (sets the mock cuFile library first)
from elbencho_b200 import BenchPhase, WorkerConfig, WorkerError, WorkerManager  # noqa: E402
from elbencho_b200 import kernels  # noqa: E402
from elbencho_b200.worker import IOEngine, PathType  # noqa: E402
from tests import cdc_model as model  # noqa: E402
from tests import reduce_model, tree_model  # noqa: E402
from tests.test_compress_stats import make_data  # noqa: E402
from tests.test_custom_tree_gpu import TREE_TEXT  # noqa: E402
from tests.test_checksums_gpu import make_workdir, run_cli  # noqa: E402
from tests.test_reduce_stats_gpu import Table, _pinned_descs, workdir  # noqa: E402,F401

pytestmark = pytest.mark.gpu

KiB, MiB, GiB = 1 << 10, 1 << 20, 1 << 30


def _slots(lengths, avg):
    return max(1, max((n + avg // 4 - 1) // (avg // 4) for n in lengths))


def _launch(blocks, avg, table, stream=None, slots=None):
    """blocks: [(device tensor, byte offset, length)]: the cut and the hash-insert on one stream
    -> (descs, counts, ends, digests) tensors"""
    slots = slots or _slots([n for _, _, n in blocks], avg)
    descs = _pinned_descs([(t, o, n, 0) for t, o, n in blocks])
    counts = torch.full((len(blocks),), -1, dtype=torch.int32, device="cuda")
    ends = torch.zeros(len(blocks) * slots, dtype=torch.int64, device="cuda")
    digests = torch.zeros(len(blocks) * slots * 32, dtype=torch.uint8, device="cuda")
    s = stream or torch.cuda.current_stream()
    shift = avg.bit_length() - 1
    with torch.cuda.stream(s):
        kernels.cdc_cut(descs.data_ptr(), len(blocks), shift, slots, counts.data_ptr(),
                        ends.data_ptr(), s.cuda_stream)
        kernels.cdc_hash_insert(descs.data_ptr(), len(blocks), shift, slots, counts.data_ptr(),
                                ends.data_ptr(), digests.data_ptr(), table.keys_ptr,
                                table.payloads_ptr, table.entries, table.counters.data_ptr(),
                                s.cuda_stream)
    return descs, counts, ends, digests, slots


def _place(datas, odd=True):
    buf = torch.zeros(sum(len(d) + 64 for d in datas) + 64, dtype=torch.uint8, device="cuda")
    blocks, pos = [], 0
    for i, data in enumerate(datas):
        off = pos + ((i * 7) % 5 if odd else 0)
        if data:
            buf[off:off + len(data)] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
        blocks.append((buf, off, len(data)))
        pos += len(data) + 64
    return buf, blocks


def _check_cuts_and_digests(datas, avg, launched):
    _, counts, ends, digests, slots = launched
    torch.cuda.synchronize()
    counts = counts.cpu().numpy()
    ends = ends.cpu().numpy().reshape(len(datas), slots)
    digests = digests.cpu().numpy().reshape(len(datas), slots, 32)
    for i, data in enumerate(datas):
        lengths = model.cut_lengths(data, avg) if data else []
        got = ends[i, :counts[i]].tolist()
        assert got == np.cumsum(lengths).tolist(), "descriptor %d" % i
        start = 0
        for j, end in enumerate(got):
            assert digests[i, j].tobytes() == blake3.blake3(data[start:end]).digest()
            start = end


def _table_keys(table):
    return {k: v[0] for k, v in table.stored().items()}


def _model_table(datas, avg):
    out = {}
    for data in datas:
        off = 0
        for length in (model.cut_lengths(data, avg) if data else []):
            out.setdefault(model.key(data[off:off + length]), length)
            off += length
    return out


def _ragged_datas(avg, seed):
    lo, hi = avg // 4, 4 * avg
    rnd = make_data("random", 6 * hi + 13, seed)
    return [rnd, bytes(2 * hi + 5), make_data("blockvar", 5 * hi + 7, seed + 1),
            rnd[:lo - 1], rnd[:lo], rnd[:hi], rnd[7:hi + 1000], b"", rnd[3:],
            make_data("text", 3 * hi, seed + 2), rnd[:hi] + bytes(hi)]


@pytest.mark.parametrize("avg", [4 * KiB, 16 * KiB, 256 * KiB])
@pytest.mark.parametrize("odd", [False, True], ids=["aligned", "odd"])
def test_cuts_and_digests_match_the_model(cuda_device, avg, odd):
    datas = _ragged_datas(avg, avg + odd)
    _, blocks = _place(datas, odd)
    table = Table(1 << 16)
    launched = _launch(blocks, avg, table)
    _check_cuts_and_digests(datas, avg, launched)
    want = _model_table(datas, avg)
    assert _table_keys(table) == want
    n, b = sum(len(model.cut_lengths(d, avg)) for d in datas if d), sum(map(len, datas))
    table.sum()
    chunks, nbytes, d, u, s, overflow = table.read_counters()
    assert (chunks, nbytes, d, u, s, overflow) == (n, b, len(want), sum(want.values()),
                                                  sum(want.values()), 0)


def test_many_descriptors_per_launch(cuda_device):
    avg = 16 * KiB
    rnd = make_data("random", 8 * MiB, 5)
    datas = [rnd[i * 37:i * 37 + 256 * KiB + i] for i in range(64)]
    _, blocks = _place(datas)
    table = Table(1 << 16)
    _check_cuts_and_digests(datas, avg, _launch(blocks, avg, table))
    assert _table_keys(table) == _model_table(datas, avg)


def test_block_past_4gib(cuda_device):
    """one descriptor whose window crosses 4 GiB of device memory"""
    avg = 64 * KiB
    tail = make_data("blockvar", 3 * MiB + 11, 9)
    big = torch.zeros(4 * GiB + 4 * MiB, dtype=torch.uint8, device="cuda")
    off = 4 * GiB - MiB - 3
    big[off:off + len(tail)] = torch.frombuffer(bytearray(tail), dtype=torch.uint8).cuda()
    table = Table(1 << 12)
    _check_cuts_and_digests([tail], avg, _launch([(big, off, len(tail))], avg, table))
    del big


def test_two_streams_insert_into_one_table(cuda_device):
    avg = 4 * KiB
    datas = _ragged_datas(avg, 3)
    _, blocks = _place(datas)
    table = Table(1 << 14)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    keep = [_launch(blocks, avg, table, s1), _launch(blocks, avg, table, s2)]
    torch.cuda.synchronize()
    want = _model_table(datas, avg)
    assert _table_keys(table) == want
    chunks, nbytes = table.read_counters()[:2]
    assert chunks == 2 * sum(len(model.cut_lengths(d, avg)) for d in datas if d)
    assert nbytes == 2 * sum(map(len, datas))
    del keep


def test_merge_of_two_tables(cuda_device):
    avg = 4 * KiB
    datas_a, datas_b = _ragged_datas(avg, 1), _ragged_datas(avg, 1)[:3] + _ragged_datas(avg, 2)
    _, blocks_a = _place(datas_a)
    _, blocks_b = _place(datas_b)
    table_a, table_b = Table(1 << 14), Table(1 << 14)
    keep = [_launch(blocks_a, avg, table_a), _launch(blocks_b, avg, table_b)]
    kernels.reduce_merge(table_b.keys_ptr, table_b.payloads_ptr, table_b.entries,
                         table_a.keys_ptr, table_a.payloads_ptr, table_a.entries,
                         table_a.counters.data_ptr())
    table_a.sum()
    torch.cuda.synchronize()
    want = _model_table(datas_a + datas_b, avg)
    assert _table_keys(table_a) == want
    assert table_a.read_counters()[2:4] == (len(want), sum(want.values()))
    del keep


def test_overflow_flag(cuda_device):
    avg = 4 * KiB
    datas = [make_data("random", 2 * MiB, 4)]
    _, blocks = _place(datas)
    table = Table(64)
    keep = _launch(blocks, avg, table)
    torch.cuda.synchronize()
    assert table.read_counters()[5] == 1
    assert len(table.stored()) == 64
    del keep


# ---- the worker ----------------------------------------------------------------------------

def expected_counts(paths, block_size, avg):
    datas = []
    for path in paths:
        with open(path, "rb") as f:
            datas.append(f.read())
    return model.counts(datas, block_size, avg)


def run_phases(cfg_args, phases=(BenchPhase.CREATEFILES, BenchPhase.READFILES), also=()):
    out = []
    with WorkerManager(WorkerConfig(**cfg_args)) as mgr:
        for phase in phases:
            res = mgr.run_phase(phase)
            out.append((mgr.cdc_stats(), res["num_kernel_launches"],
                        tuple(getattr(mgr, name)() for name in also)))
    return out


@pytest.mark.parametrize("content", [dict(block_variance_percent=50),
                                     dict(integrity_check_salt=11,
                                          integrity_check_kind=kernels.VERIFY_RANDOM,
                                          verify_random_grain=16 * KiB, dedupe_percent=50)],
                         ids=["var50", "dedupe50"])
@pytest.mark.parametrize("variant", [
    dict(block_size=64 * KiB), dict(block_size=256 * KiB, num_threads=8),
    dict(block_size=MiB, io_engine=IOEngine.AIO, io_depth=8),
    dict(block_size=256 * KiB, staging_engine=1), dict(block_size=256 * KiB, staging_engine=2),
    dict(block_size=256 * KiB, use_direct_io=True), dict(block_size=256 * KiB, use_cufile=True),
], ids=["b64k", "threads8", "aio8", "kernel", "copyengine", "direct", "cufile"])
def test_counts_match_the_files(variant, content, cuda_device):
    whole = variant.get("use_direct_io") or variant.get("use_cufile")
    workdir = make_workdir(direct=bool(whole))
    try:
        paths = [os.path.join(workdir, "f%d" % i) for i in range(2)]
        size = 2 * MiB + (0 if whole else 20 * KiB + 3)
        out = run_phases(dict(paths=paths, file_size=size, cdc_avg=4 * KiB, **content,
                              **variant))
        want = expected_counts(paths, variant["block_size"], 4 * KiB)
        assert out[0][0] == want and out[1][0] == want
    finally:
        shutil.rmtree(workdir, ignore_errors=True)


def test_dir_mode(workdir):
    args = dict(paths=[workdir], path_type=PathType.DIR, num_dirs=2, num_files=3,
                num_threads=2, block_size=128 * KiB, file_size=256 * KiB + 4 * KiB,
                block_variance_percent=50, cdc_avg=4 * KiB)
    out = run_phases(args, phases=(BenchPhase.CREATEDIRS, BenchPhase.CREATEFILES,
                                   BenchPhase.READFILES))[1:]
    files = [os.path.join(root, f) for root, _, names in os.walk(workdir) for f in names]
    assert len(files) == 12
    want = expected_counts(sorted(files), 128 * KiB, 4 * KiB)
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
                          tree_file_path=tree_path, cdc_avg=4 * KiB),
                     phases=(BenchPhase.CREATEDIRS, BenchPhase.CREATEFILES,
                             BenchPhase.READFILES))[1:]
    want = expected_counts([os.path.join(bench_dir, p) for p, _ in files], 64 * KiB, 4 * KiB)
    assert out[0][0] == want and out[1][0] == want


def test_shifted_copy(workdir):
    """random data R, 3 bytes, R again, read whole: CDC finds the copy, fixed-offset dedupe
    finds nothing"""
    rnd = make_data("random", 8 * MiB, 21)
    data = rnd + b"xyz" + rnd
    path = os.path.join(workdir, "f")
    with open(path, "wb") as f:
        f.write(data)
    out = run_phases(dict(paths=[path], file_size=len(data), block_size=MiB, num_threads=4,
                          cdc_avg=16 * KiB, dedupe_chunk=16 * KiB),
                     phases=(BenchPhase.READFILES,), also=("dedupe_stats",))
    (n, d, b, u), _, (dedupe,) = out[0]
    assert (n, d, b, u) == model.counts([data], MiB, 16 * KiB)
    assert 1.9 < b / u < 2.0
    assert dedupe[0] == dedupe[1]  # (N == D: no duplicate 16K chunk)


def test_two_gpus_give_the_result_of_one(workdir):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    paths = [os.path.join(workdir, "f%d" % i) for i in range(4)]
    args = dict(paths=paths, file_size=MiB, block_size=256 * KiB, num_threads=4,
                integrity_check_salt=3, integrity_check_kind=kernels.VERIFY_RANDOM,
                verify_random_grain=16 * KiB, dedupe_percent=50, cdc_avg=4 * KiB)
    one = run_phases(dict(args, gpu_ids=(0,)))
    two = run_phases(dict(args, gpu_ids=(0, 1)), phases=(BenchPhase.READFILES,))
    assert two[0][0] == one[1][0] == one[0][0] == expected_counts(paths, 256 * KiB, 4 * KiB)


def test_next_to_the_other_stats(workdir):
    """--dedupestats, --reducestats and BLAKE3 --checksums in the same run keep their own
    numbers"""
    paths = [os.path.join(workdir, "f%d" % i) for i in range(2)]
    grain = 16 * KiB
    out = run_phases(dict(paths=paths, file_size=MiB, block_size=256 * KiB,
                          integrity_check_salt=9, integrity_check_kind=kernels.VERIFY_RANDOM,
                          verify_random_grain=grain, dedupe_percent=50, cdc_avg=16 * KiB,
                          dedupe_chunk=grain, reduce_chunk=grain, checksums=True,
                          checksum_algo="blake3", checksum_chunk_shift=14),
                     also=("dedupe_stats", "reduce_stats"))
    datas = [open(p, "rb").read() for p in paths]
    want = model.counts(datas, 256 * KiB, 16 * KiB)
    want_reduce = reduce_model.counts(datas, grain)
    keys = [k for d in datas for k in reduce_model.chunk_keys(d, grain)]
    for stats, _, (dedupe, reduce) in out:
        assert stats == want
        assert reduce == want_reduce
        assert dedupe[:2] == (len(keys), len(set(keys)))


def test_launches_and_copies(workdir):
    """without --cdcstats a phase launches and copies what it did before: one fill / verify
    launch per batch, the data once each way; with it, two launches per batch more (cut,
    hash-insert) and no copy"""
    path = os.path.join(workdir, "f")
    size, block, batch_blocks = 8 * MiB, MiB, 2
    num_batches = size // block // batch_blocks
    counters = {}
    for avg in (0, 16 * KiB):
        cfg = WorkerConfig(paths=[path], file_size=size, block_size=block,
                           pipeline_batch_blocks=batch_blocks, integrity_check_salt=5,
                           staging_engine=2, cdc_avg=avg)
        with WorkerManager(cfg) as mgr:
            for phase in (BenchPhase.CREATEFILES, BenchPhase.READFILES):
                r = mgr.run_phase(phase)
                counters[avg, phase] = (r["num_kernel_launches"], r["h2d_bytes"],
                                        r["d2h_bytes"])
            if not avg:
                with pytest.raises(WorkerError, match="CDC stats are off"):
                    mgr.cdc_stats()
    assert counters[0, BenchPhase.CREATEFILES] == (num_batches, 0, size)
    assert counters[0, BenchPhase.READFILES] == (num_batches, size, 0)
    assert counters[16 * KiB, BenchPhase.CREATEFILES] == (3 * num_batches, 0, size)
    assert counters[16 * KiB, BenchPhase.READFILES] == (3 * num_batches, size, 0)


def test_setter_rejections(tmp_path, cuda_device):
    cfg = WorkerConfig(paths=[str(tmp_path / "f")], block_size=32 * KiB, file_size=4 * MiB,
                       cdc_avg=16 * KiB)
    with pytest.raises(WorkerError, match="below the largest CDC chunk"):
        WorkerManager(cfg)
    for extra, message in [(dict(use_random_offsets=True), "random offsets"),
                           (dict(rwmix_read_percent=20), "rwmix")]:
        cfg = WorkerConfig(paths=[str(tmp_path / "f")], block_size=MiB, file_size=4 * MiB,
                           cdc_avg=16 * KiB, **extra)
        with pytest.raises(WorkerError, match=message):
            WorkerManager(cfg)


def test_cli_prints_the_line(workdir):
    path = os.path.join(workdir, "f")
    res = run_cli("-w", "-r", "-t", "2", "-b", "1m", "-s", "8m", "--gpuids", "0",
                  "--verifyrand", "7", "--verifyrandgrain", "64k", "--dedupepct", "50",
                  "--cdcstats", "16k", "--dedupestats", "16k", path)
    assert res.returncode == 0, res.stderr
    lines = [line for line in res.stdout.splitlines() if line.startswith("CDC: ")]
    assert len(lines) == 2 and lines[0] == lines[1]
    n, d, b, u = expected_counts([path], MiB, 16 * KiB)
    assert lines[0] == model.line(16 * KiB, n, d, b, u)
