"""GPU tests of --dedupestats: the insert kernel against a Python set (one launch, two streams into
one table, a table at load 0.5, planted zero digests, a table too small that sets the overflow
flag, a merge of two tables), then the worker's counts against chunk digests of the files on disk
(block sizes, threads, AIO, staging engines, --direct, mock cuFile, dir mode, custom tree mode, a
short last chunk, zero files, --verify data, a shared BLAKE3 checksum launch, a list of another
algorithm between phases), counts that tests/dedupe_model.py fixes for --dedupepct data at K =
G/4, G and 2G and that block-keyed data with --blockvarpct 0 fixes, the last data set thread's
remainder, the launches and copies without the option, and the console line of the command
line."""
import os
import shutil

import pytest
import torch

from tests import test_checksums_gpu as base  # noqa: F401  (sets the mock cuFile library first)
from elbencho_b200 import BenchPhase, WorkerConfig, WorkerError, WorkerManager  # noqa: E402
from elbencho_b200 import kernels  # noqa: E402
from elbencho_b200.worker import IOEngine, PathType  # noqa: E402
from tests import blake3_model as model  # noqa: E402
from tests import dedupe_model  # noqa: E402
from tests import tree_model  # noqa: E402
from tests.test_custom_tree_gpu import TREE_TEXT  # noqa: E402
from tests.test_checksums_gpu import make_workdir, run_cli  # noqa: E402

pytestmark = pytest.mark.gpu

KiB, MiB = 1 << 10, 1 << 20


def _key(digest):
    return bytes([digest[0] | 1]) + bytes(digest[1:16])


class Table:
    def __init__(self, entries):
        self.entries = entries
        self.table = torch.zeros(entries * 16, dtype=torch.uint8, device="cuda")
        self.counters = torch.zeros(32, dtype=torch.uint8, device="cuda")

    def read(self):
        torch.cuda.synchronize()
        return kernels.dedupe_counters(self.counters.cpu().numpy().tobytes())


def _insert(table, digests, shift, chunks_per_desc, stream=None, zero=None):
    """digests: bytes of 32 per chunk, chunks_per_desc chunks per descriptor"""
    n = len(digests) // 32
    num_descs = n // chunks_per_desc
    raw = kernels.pack_block_descs([(0x1000, chunks_per_desc << shift, i << 30, 0)
                                    for i in range(num_descs)])
    descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).pin_memory()
    dev = torch.frombuffer(bytearray(digests), dtype=torch.uint8).cuda()
    s = stream or torch.cuda.current_stream()
    with torch.cuda.stream(s):
        kernels.dedupe_insert(descs.data_ptr(), num_descs, shift, chunks_per_desc, dev.data_ptr(),
                              table.table.data_ptr(), table.entries, table.counters.data_ptr(),
                              zero, s.cuda_stream)
    return descs, dev  # (kept alive until the stream is done)


def _digests(n, num_distinct, seed, zero=None, num_zero=0):
    g = torch.Generator().manual_seed(seed)
    pool = torch.randint(0, 256, (num_distinct, 32), dtype=torch.uint8, generator=g)
    pick = torch.cat([torch.arange(num_distinct), torch.randint(0, num_distinct,
                                                                 (n - num_distinct,), generator=g)])
    rows = [bytes(pool[i].numpy().tobytes()) for i in pick.tolist()]
    for i in range(num_zero):
        rows[(i * 7919) % n] = zero
    return rows


@pytest.mark.parametrize("load", [0.1, 0.5])
def test_insert_matches_a_set(cuda_device, load):
    shift, n, distinct = 12, 1 << 15, 5000
    zero = kernels.dedupe_zero_digest(shift)
    rows = _digests(n, distinct, 1, zero, 300)
    table = Table(1 << max(10, (int(len(set(map(_key, rows))) / load) - 1).bit_length()))
    keep = _insert(table, b"".join(rows), shift, 16)
    chunks, got_distinct, got_zero, overflow = table.read()
    del keep
    assert (chunks, got_distinct, got_zero, overflow) == (n, len(set(map(_key, rows))),
                                                         sum(r == zero for r in rows), 0)


def test_two_streams_into_one_table(cuda_device):
    shift, n = 16, 1 << 14
    rows = _digests(n, 3000, 2)
    table = Table(1 << 13)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    keep = [_insert(table, b"".join(rows[:n // 2]), shift, 4, s1),
            _insert(table, b"".join(rows[n // 2:]), shift, 4, s2)]
    assert table.read()[:3] == (n, len(set(map(_key, rows))), 0)
    del keep


def test_all_zero_key_is_an_entry(cuda_device):
    # a digest whose first 16 bytes are zero takes bit 0 like any other: it is not an empty slot
    rows = [bytes(32)] * 5 + [bytes([1]) + bytes(31)] * 3 + [bytes(16) + bytes([9]) * 16]
    table = Table(1024)
    keep = _insert(table, b"".join(rows), 12, 1)
    assert table.read() == (9, 1, 0, 0)  # (bit 0 merges them: one key)
    del keep


def test_small_table_sets_overflow_without_a_fault(cuda_device):
    rows = _digests(4096, 4096, 3)
    table = Table(1024)
    keep = _insert(table, b"".join(rows), 12, 1)
    chunks, distinct, _, overflow = table.read()
    del keep
    assert overflow == 1 and chunks == 4096 and distinct == 1024
    # the device is fine afterwards
    assert torch.ones(4, device="cuda").sum().item() == 4


def test_merge_of_two_tables(cuda_device):
    a_rows, b_rows = _digests(6000, 2000, 4), _digests(6000, 2000, 5)
    b_rows[:500] = a_rows[:500]
    a, b = Table(1 << 13), Table(1 << 12)
    keep = [_insert(a, b"".join(a_rows), 12, 1), _insert(b, b"".join(b_rows), 12, 1)]
    torch.cuda.synchronize()
    kernels.dedupe_merge(b.table.data_ptr(), b.entries, a.table.data_ptr(), a.entries,
                         a.counters.data_ptr(), torch.cuda.current_stream().cuda_stream)
    chunks, distinct, _, overflow = a.read()
    assert (chunks, overflow) == (6000, 0)
    assert distinct == len(set(map(_key, a_rows)) | set(map(_key, b_rows)))
    del keep


# ---- the worker ----------------------------------------------------------------------------

@pytest.fixture()
def workdir(cuda_device):
    path = make_workdir()
    yield path
    shutil.rmtree(path, ignore_errors=True)


def expected_counts(paths, chunk):
    """(chunks, distinct, zero) of the files' chunk digests (the `blake3` package, else the
    model)"""
    try:
        import blake3

        def chunk_digests(data):
            return [blake3.blake3(data[p:p + chunk]).digest() for p in range(0, len(data), chunk)]
    except ImportError:
        def chunk_digests(data):
            return model.chunk_digests(data, chunk)
    zero = model.digest(bytes(chunk))
    digests = []
    for path in paths:
        with open(path, "rb") as f:
            digests += chunk_digests(f.read())
    return len(digests), len(set(map(_key, digests))), sum(d == zero for d in digests)


def run_phases(cfg_args, phases=(BenchPhase.CREATEFILES, BenchPhase.READFILES)):
    out = []
    with WorkerManager(WorkerConfig(**cfg_args)) as mgr:
        for phase in phases:
            res = mgr.run_phase(phase)
            out.append((mgr.dedupe_stats(), res["num_kernel_launches"]))
    return out


CONTENT = dict(integrity_check_salt=77, integrity_check_kind=kernels.VERIFY_RANDOM,
               verify_random_grain=16 * KiB, dedupe_percent=50, block_variance_percent=100)


@pytest.mark.parametrize("variant", [
    dict(block_size=16 * KiB), dict(block_size=64 * KiB), dict(block_size=256 * KiB),
    dict(block_size=64 * KiB, num_threads=8),
    dict(block_size=64 * KiB, io_engine=IOEngine.AIO, io_depth=16),
    dict(block_size=64 * KiB, staging_engine=1), dict(block_size=64 * KiB, staging_engine=2),
    dict(block_size=64 * KiB, use_direct_io=True),
    dict(block_size=64 * KiB, use_cufile=True),
], ids=["1K", "4K", "16K", "threads8", "aio16", "kernel", "copyengine", "direct", "cufile"])
def test_counts_are_invariant(variant, cuda_device):
    whole = variant.get("use_direct_io") or variant.get("use_cufile")
    workdir = make_workdir(direct=bool(whole))
    try:
        paths = [os.path.join(workdir, "f%d" % i) for i in range(2)]
        size = 4 * MiB + (0 if whole else 20 * KiB)  # (a short last chunk unless whole blocks)
        out = run_phases(dict(paths=paths, file_size=size, dedupe_chunk=16 * KiB, **CONTENT,
                              **variant))
        want = expected_counts(paths, 16 * KiB)
        assert out[0][0] == want and out[1][0] == want
        assert want[1] < want[0]  # (--dedupepct 50: duplicate grains, K = the grain)
    finally:
        shutil.rmtree(workdir, ignore_errors=True)


def test_dir_mode(workdir):
    args = dict(paths=[workdir], path_type=PathType.DIR, num_dirs=2, num_files=3,
                num_threads=2, block_size=128 * KiB, file_size=512 * KiB + 4 * KiB,
                dedupe_chunk=4 * KiB, **CONTENT)
    out = run_phases(args, phases=(BenchPhase.CREATEDIRS, BenchPhase.CREATEFILES,
                                   BenchPhase.READFILES))[1:]
    files = [os.path.join(root, f) for root, _, names in os.walk(workdir) for f in names]
    assert len(files) == 12
    want = expected_counts(sorted(files), 4 * KiB)
    assert out[0][0] == want and out[1][0] == want


def test_verify_data_is_all_distinct(workdir):
    path = os.path.join(workdir, "f")
    out = run_phases(dict(paths=[path], file_size=8 * MiB, block_size=MiB,
                          integrity_check_salt=5, dedupe_chunk=4 * KiB))
    assert out[0][0] == (2048, 2048, 0) and out[1][0] == (2048, 2048, 0)


def test_zero_file_with_a_short_last_chunk(workdir):
    path = os.path.join(workdir, "zeros")
    with open(path, "wb") as f:
        f.write(bytes(3 * MiB + 4 * KiB))
    out = run_phases(dict(paths=[path], file_size=3 * MiB + 4 * KiB, block_size=MiB,
                          dedupe_chunk=64 * KiB), phases=(BenchPhase.READFILES,))
    assert out[0][0] == (49, 2, 48)  # (the 4 KiB tail is a chunk of its own, not a zero chunk)


def test_shared_blake3_launch_keeps_the_list(workdir):
    paths = [os.path.join(workdir, "f%d" % i) for i in range(2)]
    common = dict(paths=paths, file_size=2 * MiB, block_size=256 * KiB, checksums=True,
                  checksum_algo="blake3", checksum_chunk_shift=16, **CONTENT)
    with WorkerManager(WorkerConfig(**common)) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
        plain = mgr.run_phase(BenchPhase.READFILES)
        plain_list = mgr.checksums_text()
    with WorkerManager(WorkerConfig(dedupe_chunk=64 * KiB, **common)) as mgr:
        res = mgr.run_phase(BenchPhase.READFILES)
        assert mgr.checksums_text() == plain_list
        assert mgr.dedupe_stats() == expected_counts(paths, 64 * KiB)
    # one BLAKE3 launch per batch: the insert is the only launch added
    batches = plain["num_kernel_launches"] // 2
    assert res["num_kernel_launches"] == plain["num_kernel_launches"] + batches


def test_list_of_another_algorithm_between_phases(workdir):
    paths = [os.path.join(workdir, "f%d" % i) for i in range(2)]
    common = dict(paths=paths, file_size=2 * MiB, block_size=256 * KiB, **CONTENT)
    with WorkerManager(WorkerConfig(checksums=True, checksum_algo="crc32c",
                                    checksum_chunk_shift=16, **common)) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
        text = "# phase WRITE chunk 65536 crc32c\n" + mgr.checksums_text()
    want = expected_counts(paths, 64 * KiB)
    with WorkerManager(WorkerConfig(dedupe_chunk=64 * KiB, **common)) as mgr:
        mgr.run_phase(BenchPhase.READFILES)
        assert mgr.dedupe_stats() == want
        mgr.set_checksum_list(text)
        mgr.run_phase(BenchPhase.READFILES)
        assert mgr.dedupe_stats() == want


def test_clean_path_costs_nothing(workdir):
    """without --dedupestats a phase launches and copies what it did before: one fill / verify
    launch per batch, the data once each way; with it, a BLAKE3 launch and an insert per batch
    more and no copy"""
    path = os.path.join(workdir, "f")
    size, block, batch_blocks = 8 * MiB, MiB, 2
    num_batches = size // block // batch_blocks
    counters = {}
    for dedupe in (0, 64 * KiB):
        cfg = WorkerConfig(paths=[path], file_size=size, block_size=block,
                           pipeline_batch_blocks=batch_blocks, integrity_check_salt=5,
                           staging_engine=2, dedupe_chunk=dedupe)
        with WorkerManager(cfg) as mgr:
            for phase in (BenchPhase.CREATEFILES, BenchPhase.READFILES):
                r = mgr.run_phase(phase)
                counters[dedupe, phase] = (r["num_kernel_launches"], r["h2d_bytes"],
                                           r["d2h_bytes"])
            if not dedupe:
                with pytest.raises(WorkerError, match="dedupe stats are off"):
                    mgr.dedupe_stats()
    assert counters[0, BenchPhase.CREATEFILES] == (num_batches, 0, size)
    assert counters[0, BenchPhase.READFILES] == (num_batches, size, 0)
    assert counters[64 * KiB, BenchPhase.CREATEFILES] == (3 * num_batches, 0, size)
    assert counters[64 * KiB, BenchPhase.READFILES] == (3 * num_batches, size, 0)


# ---- counts that the data generator's model fixes ------------------------------------------

SEED, GRAIN = 41, 16 * KiB


@pytest.mark.parametrize("dedupe_pct", [0, 50, 100])
def test_grain_data_counts_match_the_model(workdir, dedupe_pct):
    """--verifyrand --verifyrandgrain G --dedupepct P over two files: at K = G the distinct chunks
    are tests/dedupe_model.py's distinct grains, at K = G/4 four times as many (the quarters of a
    random grain differ), at K = 2G the distinct pairs of the model's grain keys"""
    paths = [os.path.join(workdir, "f0"), os.path.join(workdir, "f1")]
    size = 4 * MiB
    grain_shift = GRAIN.bit_length() - 1
    grains = [(key, g * GRAIN) for key in range(len(paths)) for g in range(size // GRAIN)]
    keys = {(key, off): dedupe_model.grain_key(SEED, key, off, grain_shift, dedupe_pct)
            for key, off in grains}
    distinct = dedupe_model.distinct_grains(grains, dedupe_pct)
    pairs = len({(keys[key, off], keys[key, off + GRAIN]) for key, off in grains
                 if off % (2 * GRAIN) == 0})
    want = {GRAIN // 4: (4 * len(grains), 4 * distinct, 0), GRAIN: (len(grains), distinct, 0),
            2 * GRAIN: (len(grains) // 2, pairs, 0)}
    content = dict(integrity_check_salt=SEED, integrity_check_kind=kernels.VERIFY_RANDOM,
                   verify_random_grain=GRAIN, dedupe_percent=dedupe_pct,
                   block_variance_percent=100)
    for chunk in (GRAIN, GRAIN // 4, 2 * GRAIN):
        out = run_phases(dict(paths=paths, file_size=size, block_size=128 * KiB, num_threads=3,
                              dedupe_chunk=chunk, **content))
        assert out[0][0] == want[chunk] and out[1][0] == want[chunk], chunk
    if dedupe_pct == 0:
        assert distinct == len(grains)
    if dedupe_pct == 100:
        assert distinct < len(grains)


def test_zero_variance_blocks_are_one_chunk_each(workdir):
    """--verifyrand --blockvarpct 0 -b 1M: a block is one 8-byte value repeated, so its 16 chunks
    of 64 KiB are identical and the blocks differ"""
    path = os.path.join(workdir, "f")
    size = 8 * MiB
    out = run_phases(dict(paths=[path], file_size=size, block_size=MiB,
                          integrity_check_salt=SEED, integrity_check_kind=kernels.VERIFY_RANDOM,
                          block_variance_percent=0, dedupe_chunk=64 * KiB))
    want = (size // (64 * KiB), size // MiB, 0)
    assert out[0][0] == want and out[1][0] == want
    assert expected_counts([path], 64 * KiB) == want


def test_last_data_set_thread_takes_the_remainder(workdir):
    """one 31 MiB file of 1 MiB blocks over 16 data set threads, of which this process runs the
    last (--rankoffset 15): that worker moves its standard block plus the remainder, 16 blocks of
    256 distinct 4 KiB chunks, and its table is sized for them"""
    path = os.path.join(workdir, "f")
    out = run_phases(dict(paths=[path], file_size=31 * MiB, block_size=MiB, num_threads=1,
                          rank_offset=15, num_dataset_threads=16, integrity_check_salt=5,
                          dedupe_chunk=4 * KiB))
    assert out[0][0] == (4096, 4096, 0) and out[1][0] == (4096, 4096, 0)


def test_custom_tree_mode(workdir):
    """custom tree mode: files of many sizes (empty, one byte, short last chunks), three threads"""
    tree_path = os.path.join(workdir, "tree.txt")
    bench_dir = os.path.join(workdir, "bench")
    os.mkdir(bench_dir)
    with open(tree_path, "w") as f:
        f.write(TREE_TEXT)
    _, files = tree_model.parse_tree(TREE_TEXT)
    out = run_phases(dict(paths=[bench_dir], path_type=PathType.DIR, num_threads=3,
                          block_size=64 * KiB, block_variance_percent=40,
                          tree_file_path=tree_path, dedupe_chunk=16 * KiB),
                     phases=(BenchPhase.CREATEDIRS, BenchPhase.CREATEFILES,
                             BenchPhase.READFILES))[1:]
    want = expected_counts([os.path.join(bench_dir, p) for p, _ in files], 16 * KiB)
    assert want[0] == sum(-(-size // (16 * KiB)) for _, size in files)
    assert out[0][0] == want and out[1][0] == want


def test_two_gpus_count_as_one(workdir):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    paths = [os.path.join(workdir, "f%d" % i) for i in range(4)]
    args = dict(paths=paths, file_size=2 * MiB, block_size=256 * KiB, num_threads=4,
                dedupe_chunk=16 * KiB, **CONTENT)
    one = run_phases(dict(args, gpu_ids=(0,)))
    two = run_phases(dict(args, gpu_ids=(0, 1)), phases=(BenchPhase.READFILES,))
    assert two[0][0] == one[1][0] == expected_counts(paths, 16 * KiB)


def test_cli_prints_the_line(workdir):
    path = os.path.join(workdir, "f")
    res = run_cli("-w", "-r", "-b", "1m", "-s", "8m", "--gpuids", "0", "--verifyrand", "9",
                  "--verifyrandgrain", "64k", "--dedupepct", "100", "--dedupestats", "64k", path)
    assert res.returncode == 0, res.stderr
    lines = [line for line in res.stdout.splitlines() if line.startswith("Dedupe: ")]
    assert len(lines) == 2 and lines[0] == lines[1]
    n, d = 128, expected_counts([path], 64 * KiB)[1]
    assert lines[0] == "Dedupe: %d chunks of 65536, %d distinct, 0 zero: %.2f:1" % (n, d, n / d)
