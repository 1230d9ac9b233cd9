"""GPU tests of --cdcreducestats: the cut, the hash-insert with marks and the LZ4 launch fill a
reduce table with exactly the distinct chunks of tests/cdc_reduce_model.py and their stored sizes
(random, --blockvarpct 50, zero and --dedupepct 50 data; AVG 4K, 16K, 64K and 256K; odd
addresses; a chunk that starts past 4 GiB inside a block; two streams into one table; the merge of
two tables; the sum; the overflow flag); then the worker's (N, D, B, U, S) against the model applied
to the files on disk in file and dir mode, sync and AIO, both staging engines, write then read;
the sharing of one table and one set of launches with --cdcstats at the same AVG; launches and
copies without the option; and the console line of the README's shifted-copy example."""
import os
import types

import numpy as np
import pytest
import torch

from tests import test_checksums_gpu as base  # noqa: F401  (sets the mock cuFile library first)
from elbencho_b200 import BenchPhase, WorkerConfig, WorkerError, WorkerManager  # noqa: E402
from elbencho_b200 import kernels  # noqa: E402
from elbencho_b200.worker import IOEngine, PathType  # noqa: E402
from tests import cdc_model, compress_model, reduce_model  # noqa: E402
from tests import cdc_reduce_model as model  # noqa: E402
from tests import verify_random_grain_model as grain_model  # noqa: E402
from tests.test_cdc_stats_gpu import _place, _slots  # noqa: E402
from tests.test_compress_stats import make_data  # noqa: E402
from tests.test_checksums_gpu import run_cli  # noqa: E402
from tests.test_reduce_stats_gpu import Table, _pinned_descs, workdir  # noqa: E402,F401

pytestmark = pytest.mark.gpu

KiB, MiB, GiB = 1 << 10, 1 << 20, 1 << 30


def _launch(blocks, avg, table, stream=None, slots=None):
    """blocks: [(device tensor, byte offset, length)]: the cut, the hash-insert with marks and the
    LZ4 launch on one stream -> (descs, counts, ends, marks) tensors"""
    slots = slots or _slots([n for _, _, n in blocks], avg)
    descs = _pinned_descs([(t, o, n, 0) for t, o, n in blocks])
    counts = torch.full((len(blocks),), -1, dtype=torch.int32, device="cuda")
    ends = torch.zeros(len(blocks) * slots, dtype=torch.int64, device="cuda")
    marks = torch.full((len(blocks) * slots,), 7, dtype=torch.int64, device="cuda")
    s = stream or torch.cuda.current_stream()
    shift = avg.bit_length() - 1
    with torch.cuda.stream(s):
        kernels.cdc_cut(descs.data_ptr(), len(blocks), shift, slots, counts.data_ptr(),
                        ends.data_ptr(), s.cuda_stream)
        _insert_and_compress(descs, len(blocks), shift, slots, counts, ends, marks, table, s)
    return descs, counts, ends, marks


def _insert_and_compress(descs, num_descs, shift, slots, counts, ends, marks, table, s):
    kernels.cdc_hash_insert_marks(descs.data_ptr(), num_descs, shift, slots, counts.data_ptr(),
                                  ends.data_ptr(), 0, table.keys_ptr, table.payloads_ptr,
                                  table.entries, table.counters.data_ptr(), marks.data_ptr(),
                                  s.cuda_stream)
    kernels.cdc_lz4(descs.data_ptr(), num_descs, shift, slots, counts.data_ptr(), ends.data_ptr(),
                    marks.data_ptr(), table.payloads_ptr, s.cuda_stream)


def _stored(pieces):
    """{key: (length, min(LZ4 size, length))} of the distinct pieces"""
    out = {}
    for piece in pieces:
        key = cdc_model.key(piece)
        if key not in out:
            out[key] = (len(piece), min(compress_model.size(piece), len(piece)))
    return out


def _model_stored(datas, avg):
    return model.distinct([d for d in datas if d], 1 << 62, avg)[2]


def _dedupe_data(n, seed):
    """--dedupepct 50 file content with 16 KiB grains, about half of them random"""
    return grain_model.file_content(n, 16 * KiB, 50, seed, 1, dedupe_pct=50)


def _datas(avg, seed):
    lo, hi = avg // 4, 4 * avg
    rnd = make_data("random", 6 * hi + 13, seed)
    var = make_data("blockvar", 5 * hi + 7, seed + 1)
    return [rnd, bytes(2 * hi + 5), var, rnd[:lo - 1], rnd[:hi], b"", var[3:], rnd[:hi] + var,
            _dedupe_data(6 * hi + 4099, seed + 2)]


def _check(table, datas, avg):
    want = _model_stored(datas, avg)
    table.sum()
    torch.cuda.synchronize()
    assert table.stored() == want
    n = sum(len(cdc_model.cut_lengths(d, avg)) for d in datas if d)
    u = sum(v[0] for v in want.values())
    s = sum(v[1] for v in want.values())
    assert table.read_counters() == (n, sum(map(len, datas)), len(want), u, s, 0)
    return want


@pytest.mark.parametrize("avg", [4 * KiB, 16 * KiB, 64 * KiB, 256 * KiB])
@pytest.mark.parametrize("odd", [False, True], ids=["aligned", "odd"])
def test_table_holds_the_model(cuda_device, avg, odd):
    datas = _datas(avg, avg + odd)
    _, blocks = _place(datas, odd)
    table = Table(1 << 16)
    _, counts, ends, marks = _launch(blocks, avg, table)
    want = _check(table, datas, avg)
    # one slot marked per distinct chunk, the entry its key took; the others not new
    slots = len(marks) // len(datas)
    counts, marks = counts.cpu().numpy(), marks.cpu().numpy().view(np.uint64).reshape(-1, slots)
    taken = [int(e) for i in range(len(datas)) for e in marks[i, :counts[i]]
             if e != kernels.REDUCE_NOT_NEW]
    assert len(taken) == len(set(taken)) == len(want)
    assert all(int(marks[i, j]) == 7 for i in range(len(datas)) for j in range(counts[i], slots))
    assert {table.keys()[e].tobytes() for e in taken} == set(want)


def test_random_data_does_not_shrink(cuda_device):
    avg = 16 * KiB
    datas = [make_data("random", 4 * MiB + 9, 31)]
    _, blocks = _place(datas)
    table = Table(1 << 12)
    keep = _launch(blocks, avg, table)
    want = _check(table, datas, avg)
    assert all(length == stored for length, stored in want.values())
    del keep


def test_chunk_past_4gib_in_a_block(cuda_device):
    """one descriptor of 4 GiB + 3 MiB at an odd address: 1 MiB chunks of zeros up to 4 GiB, a
    5-byte chunk of zeros, then the chunks of --blockvarpct 50 data from 4 GiB + 5 on (the ends
    given, not cut)"""
    avg = 256 * KiB
    length = 4 * GiB + 3 * MiB
    tail = make_data("blockvar", length - 4 * GiB - 5, 9)
    big = torch.zeros(length + 64, dtype=torch.uint8, device="cuda")
    big[1 + 4 * GiB + 5:1 + length] = torch.frombuffer(bytearray(tail), dtype=torch.uint8).cuda()
    tail_lengths = cdc_model.cut_lengths(tail, avg)
    chunk_ends = [(j + 1) * MiB for j in range(4096)] + [4 * GiB + 5]
    chunk_ends += (4 * GiB + 5 + np.cumsum(tail_lengths)).tolist()
    slots = _slots([length], avg)
    descs = _pinned_descs([(big, 1, length, 0)])
    counts = torch.tensor([len(chunk_ends)], dtype=torch.int32, device="cuda")
    ends = torch.zeros(slots, dtype=torch.int64, device="cuda")
    ends[:len(chunk_ends)] = torch.tensor(chunk_ends, dtype=torch.int64)
    marks = torch.zeros(slots, dtype=torch.int64, device="cuda")
    table = Table(1 << 10)
    _insert_and_compress(descs, 1, 18, slots, counts, ends, marks, table,
                         torch.cuda.current_stream())
    table.sum()
    torch.cuda.synchronize()
    pieces, start = [bytes(MiB), bytes(5)], 0
    for n in tail_lengths:
        pieces.append(tail[start:start + n])
        start += n
    want = _stored(pieces)
    assert table.stored() == want
    assert table.read_counters() == (len(chunk_ends), length, len(want),
                                     sum(v[0] for v in want.values()),
                                     sum(v[1] for v in want.values()), 0)
    del big


def test_two_streams_insert_into_one_table(cuda_device):
    avg = 4 * KiB
    datas = _datas(avg, 3)
    _, blocks = _place(datas)
    table = Table(1 << 14)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    keep = [_launch(blocks, avg, table, s1), _launch(blocks, avg, table, s2)]
    torch.cuda.synchronize()
    table.sum()
    torch.cuda.synchronize()
    want = _model_stored(datas, avg)
    assert table.stored() == want
    chunks, nbytes, d, u, s = table.read_counters()[:5]
    assert chunks == 2 * sum(len(cdc_model.cut_lengths(x, avg)) for x in datas if x)
    assert (nbytes, d) == (2 * sum(map(len, datas)), len(want))
    assert (u, s) == (sum(v[0] for v in want.values()), sum(v[1] for v in want.values()))
    del keep


def _merge(table_a, table_b, stream=0):
    kernels.reduce_merge(table_b.keys_ptr, table_b.payloads_ptr, table_b.entries,
                         table_a.keys_ptr, table_a.payloads_ptr, table_a.entries,
                         table_a.counters.data_ptr(), stream)


def test_merge_of_two_tables_carries_the_stored_sizes(cuda_device):
    avg = 16 * KiB
    datas_a, datas_b = _datas(avg, 1), _datas(avg, 1)[:3] + _datas(avg, 2)
    _, blocks_a = _place(datas_a)
    _, blocks_b = _place(datas_b)
    table_a, table_b = Table(1 << 14), Table(1 << 12)
    keep = [_launch(blocks_a, avg, table_a), _launch(blocks_b, avg, table_b)]
    _merge(table_a, table_b)
    table_a.sum()
    torch.cuda.synchronize()
    want = _model_stored(datas_a + datas_b, avg)
    assert table_a.stored() == want
    assert table_a.read_counters()[2:5] == (len(want), sum(v[0] for v in want.values()),
                                            sum(v[1] for v in want.values()))
    del keep


def test_peer_merge_of_two_gpus(cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    avg = 16 * KiB
    datas_a, datas_b = _datas(avg, 5), _datas(avg, 5)[:2] + _datas(avg, 6)
    _, blocks_a = _place(datas_a)
    table_a = Table(1 << 14)
    keep = [_launch(blocks_a, avg, table_a)]
    with torch.cuda.device(1):
        _, blocks_b = _place(datas_b)
        table_b = Table(1 << 14)
        keep.append(_launch(blocks_b, avg, table_b))
        torch.cuda.synchronize()
    piece = torch.empty(table_b.mem.numel(), dtype=torch.uint8, device="cuda:0")
    piece.copy_(table_b.mem)  # (peer to peer, as the manager copies)
    _merge(table_a, types.SimpleNamespace(keys_ptr=piece.data_ptr(),
                                          payloads_ptr=piece.data_ptr() + 16 * table_b.entries,
                                          entries=table_b.entries))
    table_a.sum()
    torch.cuda.synchronize()
    assert table_a.stored() == _model_stored(datas_a + datas_b, avg)
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

def expected_counts(paths, block_size, avg, size=None):
    datas = []
    for path in paths:
        with open(path, "rb") as f:
            datas.append(f.read(size) if size else f.read())
    return model.counts(datas, block_size, avg)


def run_phases(cfg_args, phases=(BenchPhase.CREATEFILES, BenchPhase.READFILES), also=()):
    out = []
    with WorkerManager(WorkerConfig(**cfg_args)) as mgr:
        for phase in phases:
            res = mgr.run_phase(phase)
            out.append((mgr.cdc_reduce_stats(), res["num_kernel_launches"],
                        tuple(getattr(mgr, name)() for name in also)))
    return out


@pytest.mark.parametrize("content", [dict(block_variance_percent=50),
                                     dict(integrity_check_salt=11,
                                          integrity_check_kind=kernels.VERIFY_RANDOM,
                                          verify_random_grain=16 * KiB, dedupe_percent=50)],
                         ids=["var50", "dedupe50"])
@pytest.mark.parametrize("variant", [
    dict(block_size=256 * KiB, num_threads=4),
    dict(block_size=MiB, io_engine=IOEngine.AIO, io_depth=8),
    dict(block_size=256 * KiB, staging_engine=1), dict(block_size=256 * KiB, staging_engine=2),
], ids=["sync", "aio8", "kernel", "copyengine"])
def test_counts_match_the_files(variant, content, workdir):
    paths = [os.path.join(workdir, "f%d" % i) for i in range(2)]
    size = 2 * MiB + 20 * KiB + 3
    out = run_phases(dict(paths=paths, file_size=size, cdc_reduce_avg=16 * KiB, **content,
                          **variant))
    want = expected_counts(paths, variant["block_size"], 16 * KiB)
    assert out[0][0] == want and out[1][0] == want


def test_dir_mode(workdir):
    args = dict(paths=[workdir], path_type=PathType.DIR, num_dirs=2, num_files=3,
                num_threads=2, block_size=128 * KiB, file_size=256 * KiB + 4 * KiB,
                block_variance_percent=50, cdc_reduce_avg=4 * KiB)
    out = run_phases(args, phases=(BenchPhase.CREATEDIRS, BenchPhase.CREATEFILES,
                                   BenchPhase.READFILES))[1:]
    files = [os.path.join(root, f) for root, _, names in os.walk(workdir) for f in names]
    assert len(files) == 12
    want = expected_counts(sorted(files), 128 * KiB, 4 * KiB)
    assert out[0][0] == want and out[1][0] == want


def test_two_gpus_give_the_result_of_one(workdir):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    paths = [os.path.join(workdir, "f%d" % i) for i in range(4)]
    args = dict(paths=paths, file_size=MiB, block_size=256 * KiB, num_threads=4,
                integrity_check_salt=3, integrity_check_kind=kernels.VERIFY_RANDOM,
                verify_random_grain=16 * KiB, dedupe_percent=50, cdc_reduce_avg=4 * KiB)
    one = run_phases(dict(args, gpu_ids=(0,)))
    two = run_phases(dict(args, gpu_ids=(0, 1)), phases=(BenchPhase.READFILES,))
    assert two[0][0] == one[1][0] == one[0][0] == expected_counts(paths, 256 * KiB, 4 * KiB)


def _launches_and_copies(path, **stats):
    size, block, batch_blocks = 8 * MiB, MiB, 2
    cfg = WorkerConfig(paths=[path], file_size=size, block_size=block,
                       pipeline_batch_blocks=batch_blocks, integrity_check_salt=5,
                       staging_engine=2, **stats)
    out = {}
    with WorkerManager(cfg) as mgr:
        for phase in (BenchPhase.CREATEFILES, BenchPhase.READFILES):
            r = mgr.run_phase(phase)
            out[phase] = (r["num_kernel_launches"], r["h2d_bytes"], r["d2h_bytes"],
                          mgr.cdc_stats() if stats.get("cdc_avg") else None,
                          mgr.cdc_reduce_stats() if stats.get("cdc_reduce_avg") else None)
        if not stats.get("cdc_reduce_avg"):
            with pytest.raises(WorkerError, match="CDC reduce stats are off"):
                mgr.cdc_reduce_stats()
    return out


def test_launches_copies_and_sharing_with_cdcstats(workdir):
    """without the option a phase launches and copies what it did before (one fill / verify
    launch per batch, the data once each way); with it, three launches per batch more (cut,
    hash-insert, LZ4) and no copy; with --cdcstats at the same AVG no more than that, and the
    same N, D, B and U; at another AVG both keep their own launches"""
    path = os.path.join(workdir, "f")
    nb, size = 4, 8 * MiB
    runs = {name: _launches_and_copies(path, **stats) for name, stats in [
        ("none", {}), ("cdc", dict(cdc_avg=16 * KiB)), ("reduce", dict(cdc_reduce_avg=16 * KiB)),
        ("same", dict(cdc_avg=16 * KiB, cdc_reduce_avg=16 * KiB)),
        ("other", dict(cdc_avg=4 * KiB, cdc_reduce_avg=16 * KiB))]}
    for name, extra in [("none", 0), ("cdc", 2), ("reduce", 3), ("same", 3), ("other", 5)]:
        assert runs[name][BenchPhase.CREATEFILES][:3] == ((1 + extra) * nb, 0, size), name
        assert runs[name][BenchPhase.READFILES][:3] == ((1 + extra) * nb, size, 0), name
    want = expected_counts([path], MiB, 16 * KiB)
    for phase in (BenchPhase.CREATEFILES, BenchPhase.READFILES):
        cdc, reduce = runs["same"][phase][3:]
        assert reduce == want and cdc == want[:4] == runs["cdc"][phase][3]
        assert runs["reduce"][phase][4] == want
        cdc, reduce = runs["other"][phase][3:]
        assert reduce == want
        assert cdc == cdc_model.counts([open(path, "rb").read()], MiB, 4 * KiB)


def test_setter_rejections(tmp_path, cuda_device):
    cfg = WorkerConfig(paths=[str(tmp_path / "f")], block_size=32 * KiB, file_size=4 * MiB,
                       cdc_reduce_avg=16 * KiB)
    with pytest.raises(WorkerError, match=r"below the largest CDC chunk \(--cdcreducestats\)"):
        WorkerManager(cfg)
    for extra, message in [(dict(use_random_offsets=True), "random offsets"),
                           (dict(rwmix_read_percent=20), "rwmix")]:
        cfg = WorkerConfig(paths=[str(tmp_path / "f")], block_size=MiB, file_size=4 * MiB,
                           cdc_reduce_avg=16 * KiB, **extra)
        with pytest.raises(WorkerError, match=r"CDC reduce stats \(--cdcreducestats\) .*" +
                           message):
            WorkerManager(cfg)


def test_cli_write_and_read_print_the_same_line(workdir):
    path = os.path.join(workdir, "f")
    res = run_cli("-w", "-r", "-t", "2", "-b", "1m", "-s", "8m", "--gpuids", "0",
                  "--blockvarpct", "50", "--cdcreducestats", "16k", path)
    assert res.returncode == 0, res.stderr
    lines = [line for line in res.stdout.splitlines() if line.startswith("CDC reduce: ")]
    assert len(lines) == 2 and lines[0] == lines[1]
    assert lines[0] == model.line(16 * KiB, *expected_counts([path], MiB, 16 * KiB))


def test_cli_shifted_copy(workdir):
    """the README example: a --blockvarpct 50 file and its copy behind a 3-byte header, read with
    fixed 16K and content-defined 16K chunks"""
    a, b = os.path.join(workdir, "a"), os.path.join(workdir, "b")
    res = run_cli("-w", "-t", "4", "-b", "1m", "-s", "8m", "--gpuids", "0", "--blockvarpct", "50",
                  a)
    assert res.returncode == 0, res.stderr
    with open(a, "rb") as f:
        data = f.read()
    with open(b, "wb") as f:
        f.write(b"xyz" + data)
    res = run_cli("-r", "-t", "4", "-b", "1m", "-s", "8m", "--gpuids", "0", "--reducestats", "16k",
                  "--cdcreducestats", "16k", a, b)
    assert res.returncode == 0, res.stderr
    lines = res.stdout.splitlines()
    want = expected_counts([a, b], MiB, 16 * KiB, size=8 * MiB)
    assert model.line(16 * KiB, *want) in lines
    fixed = reduce_model.counts([data, (b"xyz" + data)[:8 * MiB]], 16 * KiB)
    assert reduce_model.line(16 * KiB, *fixed) in lines
    # the copy adds about nothing to the distinct bytes of content-defined chunks (a chunk or two
    # per block edge), and as much again to those of fixed chunks
    assert want[3] < 1.25 * model.counts([data], MiB, 16 * KiB)[3]
    assert fixed[3] > 1.9 * reduce_model.counts([data], 16 * KiB)[3]
