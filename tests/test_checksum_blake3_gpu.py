"""GPU tests of the BLAKE3 kernel (elb_blake3_chunks) against the numpy model
(tests/blake3_model.py) and the goldens: whole-file runs and digests, K-chunk digests at 4 KiB,
64 KiB and 1 MiB, every length class around 64 B and 1 KiB as file tails, whole-file descriptors
of at most and more than 1 KiB, non-power-of-two blocks joined into a file's digest, odd device
addresses, ragged windows, file offsets past 4 TiB and a block past 4 GiB. Then the worker: lists
and whole-file digests in file, dir and custom tree mode; one digest across block sizes, threads,
queue depths, staging engines, --direct and mock cuFile; '-' for a --datasetthreads slice; clean
sequential, random and --infloop reads against a list; the text of a flipped byte; lists that
switch algorithms between reads; launches and copies equal to crc32's; and the command line."""
import json
import os
import random
import shutil

import numpy as np
import pytest
import torch

from tests import test_checksums_gpu as base  # noqa: F401  (sets the mock cuFile library first)
from elbencho_b200 import BenchPhase, WorkerConfig, WorkerError, WorkerManager  # noqa: E402
from elbencho_b200 import kernels  # noqa: E402
from elbencho_b200.worker import IOEngine, PathType  # noqa: E402
from tests import blake3_model as model  # noqa: E402
from tests import crc_algo_model as crc_model  # noqa: E402
from tests.test_checksums_gpu import make_workdir, run_cli, setup_mode  # noqa: E402

pytestmark = pytest.mark.gpu

KiB, MiB, GiB, TiB = 1 << 10, 1 << 20, 1 << 30, 1 << 40

LENGTHS = [1, 63, 64, 65, 127, 128, 129, 1023, 1024, 1025, 2047, 2048, 2049, 3072, 3073, 4095,
           4096, 4097, 8191, 8193, 65535, 65537, 524288, 524289, 1048575, 1048577]

with open(os.path.join(os.path.dirname(__file__), "golden", "blake3_vectors.json")) as _f:
    GOLDEN = {v["length"]: v["digest"] for v in json.load(_f)["vectors"]}


def run_blake3(blocks, shift, slots, shifts=None, launches=1):
    """blocks: [(device address, length, file offset)]; the slots of each descriptor, 32 bytes
    each, as the last of `launches` launches published them to pinned memory"""
    n = len(blocks)
    stream = torch.cuda.current_stream().cuda_stream
    raw = kernels.pack_block_descs([(ptr, length, off, 0) for ptr, length, off in blocks])
    descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).pin_memory()
    shift_arr = torch.tensor(shifts or [0] * n, dtype=torch.int64).pin_memory()
    dev = torch.zeros(max(n * slots, 1) * 32, dtype=torch.uint8, device="cuda")
    host = torch.full((max(n * slots, 1) * 32,), 0x77, dtype=torch.uint8).pin_memory()
    ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
    for _ in range(launches):
        kernels.blake3_chunks(descs.data_ptr(), shift_arr.data_ptr() if shift == 64 else 0, n,
                              shift, slots, dev.data_ptr(), host.data_ptr(), ticket.data_ptr(),
                              stream)
    torch.cuda.synchronize()
    out = host.numpy().tobytes()
    assert int(ticket.item()) == 0
    return [[out[(i * slots + j) * 32:(i * slots + j + 1) * 32] for j in range(slots)]
            for i in range(n)]


def expected(data, offset, shift, slots, is_whole_file=False):
    """the slots of a descriptor over data at file offset offset"""
    if shift == 64:
        if is_whole_file:
            want = [model.digest(data)]
        else:
            first = offset // KiB
            runs = model.canonical_runs(first, first + -(-len(data) // KiB))
            want = [model.run_cv(data[(f - first) * KiB:(f - first + c) * KiB], f) for f, c in runs]
    else:
        want = model.chunk_digests(data, 1 << shift)
    return want + [None] * (slots - len(want))


def check(got, want):
    for j, w in enumerate(want):
        if w is not None:
            assert got[j].hex() == w.hex(), j


def slots_for(length, offset, shift):
    if shift == 64:
        first = offset // KiB
        return max(1, len(model.canonical_runs(first, first + -(-length // KiB))))
    return max(1, -(-length // (1 << shift)))


@pytest.fixture(scope="module")
def buf(cuda_device):
    gen = torch.Generator("cuda").manual_seed(7)
    return torch.randint(0, 256, (16 * MiB,), dtype=torch.uint8, device="cuda", generator=gen)


@pytest.mark.parametrize("misalign", [0, 1, 5])
@pytest.mark.parametrize("shift", [64, 12, 16, 20])
def test_length_classes_as_file_tails(buf, shift, misalign):
    host = buf.cpu().numpy().tobytes()
    blocks, shifts, wants = [], [], []
    stride = 2 * MiB
    for i, length in enumerate(LENGTHS[:-2] if shift == 64 else LENGTHS):
        offset = (3 << 20) if shift < 64 else (i % 4) * 4 * MiB  # block-aligned file offsets
        src = (i * 4099 * 16) % (16 * MiB - stride) + misalign
        blocks.append((buf.data_ptr() + src, length, offset))
        shifts.append(0)
        wants.append(host[src:src + length])
    slots = max(slots_for(length, off, shift) for _, length, off in blocks)
    got = run_blake3(blocks, shift, slots, shifts)
    for i, (_, length, off) in enumerate(blocks):
        check(got[i], expected(wants[i], off, shift, slots, is_whole_file=(off == 0)))


@pytest.mark.parametrize("length", [0, 1, 64, 1023, 1024, 1025, 2048, 4096, 5121, 600 * KiB,
                                    MiB, 3 * MiB + 5])
def test_whole_file_descriptor_is_the_digest(buf, length):
    (got,) = run_blake3([(buf.data_ptr() + 3, length, 0)], 64, 1, [0])
    data = buf[3:3 + length].cpu().numpy().tobytes()
    assert got[0] == model.digest(data)


@pytest.mark.parametrize("length", sorted(GOLDEN))
def test_whole_file_goldens(cuda_device, length):
    data = model.pattern(length)
    dev = torch.frombuffer(bytearray(data) or bytearray(1), dtype=torch.uint8).cuda()
    (got,) = run_blake3([(dev.data_ptr(), length, 0)], 64, 1, [0])
    assert got[0].hex() == GOLDEN[length]


@pytest.mark.parametrize("block", [3 * KiB, 96 * KiB, 256 * KiB, MiB])
def test_blocks_join_into_the_file_digest(buf, block):
    """a file cut into blocks of the block size: the host joins the runs of all blocks"""
    size = 2 * MiB + 3 * KiB + 17
    data = buf[:size].cpu().numpy().tobytes()
    blocks = [(buf.data_ptr() + off, min(block, size - off), off) for off in range(0, size, block)]
    shifts = [size - off - length for _, length, off in blocks]
    slots = max(slots_for(length, off, 64) for _, length, off in blocks)
    got = run_blake3(blocks, 64, slots, shifts)
    runs = []
    for i, (_, length, off) in enumerate(blocks):
        first = off // KiB
        for j, (f, c) in enumerate(model.canonical_runs(first, first + -(-length // KiB))):
            runs.append((f, c, got[i][j]))
    num_chunks = -(-size // KiB)
    held = {}
    for f, c, cv in runs:  # join aligned siblings, never into the whole file
        while True:
            sib = f + c if f % (2 * c) == 0 else f - c
            if held.get(sib, (None,))[0] != c or (min(f, sib) == 0 and 2 * c == num_chunks):
                break
            _, other = held.pop(sib)
            cv = kernels.blake3_parent(*((cv, other) if sib > f else (other, cv)))
            f, c = min(f, sib), 2 * c
        held[f] = (c, cv)
    assert [(f, held[f][0]) for f in sorted(held)] == model.fold_runs(num_chunks)
    assert kernels.blake3_fold([held[f][1] for f in sorted(held)], size) == model.digest(data)


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("shift", [64, 12, 20])
def test_ragged_windows(buf, seed, shift):
    rng = random.Random(seed)
    host = buf.cpu().numpy().tobytes()
    unit = KiB if shift == 64 else 1 << shift
    blocks, shifts, wants = [], [], []
    for _ in range(rng.randrange(1, 40)):
        length = rng.choice([rng.randrange(1, 8) * unit, rng.randrange(1, 3 * MiB),
                             rng.randrange(1, 5000)])
        offset = rng.randrange(0, 64) * unit * rng.choice([1, 3, 1024])
        file_end = rng.random() < 0.5
        if not file_end:
            length = max(unit, length // unit * unit)
        src = rng.randrange(0, 16 * MiB - length - 16)
        blocks.append((buf.data_ptr() + src, length, offset))
        shifts.append(0 if file_end else rng.randrange(1, 1 << 40))
        wants.append(host[src:src + length])
    slots = max(slots_for(length, off, shift) for _, length, off in blocks)
    got = run_blake3(blocks, shift, slots, shifts, launches=2)
    for i, (_, length, off) in enumerate(blocks):
        check(got[i], expected(wants[i], off, shift, slots,
                               is_whole_file=(off == 0 and shifts[i] == 0)))


@pytest.mark.parametrize("offset", [5 * TiB, 4 * TiB + 3 * KiB, (1 << 52) + 64 * KiB])
def test_file_offsets_past_4tib(buf, offset):
    host = buf.cpu().numpy().tobytes()
    length = 200 * KiB + 7
    (got,) = run_blake3([(buf.data_ptr() + 9, length, offset)], 64,
                        slots_for(length, offset, 64), [0])
    check(got, expected(host[9:9 + length], offset, 64, len(got)))


def test_block_past_4gib(cuda_device):
    shift, length = 20, 4 * GiB + 4099
    big = torch.empty(length + 16, dtype=torch.uint8, device="cuda")
    big.random_(0, 256, generator=torch.Generator("cuda").manual_seed(5))
    ptr = big.data_ptr() + 5
    num_chunks = -(-length // (1 << shift))
    (slots,) = run_blake3([(ptr, length, 0)], shift, num_chunks)
    for j in (0, 1, 4095, 4096):
        chunk = big[5 + (j << shift):5 + min((j + 1) << shift, length)].cpu().numpy().tobytes()
        assert slots[j] == model.digest(chunk), j
    del big
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------
# worker level
# ------------------------------------------------------------------------------------------------

@pytest.fixture()
def workdir(cuda_device):
    path = make_workdir()
    yield path
    shutil.rmtree(path, ignore_errors=True)


def file_digest(path, size):
    with open(path, "rb") as f:
        data = f.read(size)
    assert len(data) == size
    return model.digest(data).hex()


def digest_lines(lines):
    """mgr.checksums() with the digests as hex (None: '-')"""
    return [(a, b, c, None if d is None else "%064x" % d) for a, b, c, d in lines]


def chunk_lines(files, shift):
    want = []
    for path in sorted(files):
        with open(path, "rb") as f:
            data = f.read(files[path])
        for off, digest in zip(range(0, files[path], 1 << shift),
                               model.chunk_digests(data, 1 << shift)):
            want.append((path, off, min(1 << shift, files[path] - off), digest.hex()))
    return want


def list_text(lines, shift, phase="WRITE"):
    return "# phase %s chunk %d blake3\n" % (phase, 1 << shift) + "".join(
        "%s %d %d %s\n" % line for line in lines)


@pytest.mark.parametrize("mode", ["file1", "file3", "dir", "tree"])
def test_lists_match_the_model(workdir, mode):
    threads = 4 if mode.startswith("file") else 3
    args, files = setup_mode(mode, workdir, threads, False)
    shift = 12 if mode == "tree" else 16
    content = {} if mode == "tree" else dict(block_variance_percent=100)
    cfg = WorkerConfig(num_threads=threads, checksums=True, checksum_chunk_shift=shift,
                       checksum_algo="blake3", **args, **content)
    with WorkerManager(cfg) as mgr:
        if args.get("path_type") == PathType.DIR:
            mgr.run_phase(BenchPhase.CREATEDIRS)
        mgr.run_phase(BenchPhase.CREATEFILES)
        written = digest_lines(mgr.checksums())
        mgr.set_checksum_list(list_text(written, shift))
        mgr.run_phase(BenchPhase.READFILES)
        read = digest_lines(mgr.checksums())
        counts = mgr.checksum_verify_counts()
    assert written == chunk_lines(files, shift)
    assert read == written
    assert counts == (len(written), len([size for size in files.values() if size]))
    cfg = WorkerConfig(num_threads=threads, checksums=True, checksum_algo="blake3", **args)
    with WorkerManager(cfg) as mgr:
        mgr.run_phase(BenchPhase.READFILES)
        lines = digest_lines(mgr.checksums())
    assert lines == [(p, files[p], files[p], file_digest(p, files[p])) for p in sorted(files)]


SHAPES = {
    "b4k_t1": dict(block_size=4 * KiB, num_threads=1),
    "b3k_t2": dict(block_size=3 * KiB, num_threads=2),
    "b96k_t3": dict(block_size=96 * KiB, num_threads=3),
    "b1m_t8": dict(block_size=MiB, num_threads=8),
    "b4m_t2": dict(block_size=4 * MiB, num_threads=2),
    "aio_qd1": dict(block_size=64 * KiB, num_threads=2, io_engine=IOEngine.AIO, io_depth=1),
    "aio_qd16": dict(block_size=64 * KiB, num_threads=4, io_engine=IOEngine.AIO, io_depth=16),
    "kernel_staging": dict(block_size=256 * KiB, num_threads=2, staging_engine=1),
    "copy_engine": dict(block_size=256 * KiB, num_threads=2, staging_engine=2),
    "cufile": dict(block_size=256 * KiB, num_threads=2, use_cufile=True),
}


@pytest.mark.parametrize("shape", list(SHAPES))
def test_whole_file_digest_is_the_same_for_every_shape(workdir, shape):
    size = 6 * MiB + 12 * KiB  # (a multiple of 3 KiB, 4 KiB and of no larger block)
    path = os.path.join(workdir, "f")
    with open(path, "wb") as f:
        f.write(np.random.default_rng(4).integers(0, 256, size, dtype=np.uint8).tobytes())
    opts = dict(SHAPES[shape])
    if opts.get("use_cufile"):
        size -= size % opts["block_size"]
    cfg = WorkerConfig(paths=[path], file_size=size, checksums=True, checksum_algo="blake3",
                       **opts)
    with WorkerManager(cfg) as mgr:
        mgr.run_phase(BenchPhase.READFILES)
        lines = digest_lines(mgr.checksums())
    assert lines == [(path, size, size, file_digest(path, size))]


def test_direct_read_digest(cuda_device):
    workdir = make_workdir(direct=True)
    try:
        path = os.path.join(workdir, "f")
        size = 4 * MiB
        with open(path, "wb") as f:
            f.write(np.random.default_rng(6).integers(0, 256, size, dtype=np.uint8).tobytes())
        cfg = WorkerConfig(paths=[path], file_size=size, block_size=256 * KiB, num_threads=4,
                           use_direct_io=True, checksums=True, checksum_algo="blake3")
        with WorkerManager(cfg) as mgr:
            mgr.run_phase(BenchPhase.READFILES)
            assert digest_lines(mgr.checksums()) == [(path, size, size, file_digest(path, size))]
    finally:
        shutil.rmtree(workdir, ignore_errors=True)


def test_dataset_thread_slice_is_incomplete(workdir):
    path = os.path.join(workdir, "f")
    size = 4 * MiB
    with open(path, "wb") as f:
        f.write(bytes(size))
    cfg = WorkerConfig(paths=[path], file_size=size, block_size=256 * KiB, num_threads=1,
                       num_dataset_threads=2, checksums=True, checksum_algo="blake3")
    with WorkerManager(cfg) as mgr:
        mgr.run_phase(BenchPhase.READFILES)
        ((p, s, covered, digest),) = digest_lines(mgr.checksums())
    assert (p, s, digest) == (path, size, None) and covered < size


def write_listed_file(workdir, size, shift, fname="f"):
    path = os.path.join(workdir, fname)
    with open(path, "wb") as f:
        f.write(np.random.default_rng(size).integers(0, 256, size, dtype=np.uint8).tobytes())
    lines = chunk_lines({path: size}, shift)
    return path, list_text(lines, shift), len(lines)


READS = {
    "seq": dict(block=4, threads=2),
    "rand": dict(block=1, threads=4, use_random_offsets=True),
    "aio_qd16_rand": dict(block=1, threads=4, io_engine=IOEngine.AIO, io_depth=16,
                          use_random_offsets=True),
    "kernel_staging": dict(block=4, threads=2, staging_engine=1),
}


@pytest.mark.parametrize("read", list(READS))
def test_clean_reads_pass(workdir, read):
    opts = dict(READS[read])
    size, shift = 4 * MiB, 16
    path, text, num_lines = write_listed_file(workdir, size, shift)
    block = opts.pop("block") << shift
    threads = opts.pop("threads")
    cfg = WorkerConfig(paths=[path], file_size=size, block_size=block, num_threads=threads,
                       rand_offset_seed=5, **opts)
    with WorkerManager(cfg) as mgr:
        mgr.set_checksum_list(text)
        res = mgr.run_phase(BenchPhase.READFILES)
        chunks, files = mgr.checksum_verify_counts()
    assert files == 1
    assert chunks == res["ops_total"]["bytes"] >> shift
    if not opts.get("use_random_offsets"):
        assert chunks == num_lines


@pytest.mark.parametrize("rand", [False, True])
def test_flipped_byte_names_its_chunk(workdir, rand):
    size, shift = 4 * MiB, 16
    path, text, _ = write_listed_file(workdir, size, shift)
    bad = 3 * MiB + 70000
    with open(path, "r+b") as f:
        f.seek(bad)
        byte = f.read(1)
        f.seek(bad)
        f.write(bytes([byte[0] ^ 0x01]))
    with open(path, "rb") as f:
        data = f.read()
    off = bad >> shift << shift
    line = next(l for l in text.splitlines() if l.startswith("%s %d " % (path, off)))
    cfg = WorkerConfig(paths=[path], file_size=size, block_size=256 * KiB, num_threads=1,
                       rand_offset_seed=3, use_random_offsets=rand)
    with WorkerManager(cfg) as mgr:
        mgr.set_checksum_list(text)
        with pytest.raises(WorkerError) as excinfo:
            mgr.run_phase(BenchPhase.READFILES)
    assert ("Checksum verification failed. File: %s; Offset: %d; Length: %d; Expected BLAKE3: %s; "
            "Actual BLAKE3: %s" % (path, off, 1 << shift, line.rsplit(" ", 1)[1],
                                    model.digest(data[off:off + (1 << shift)]).hex())
            ) in str(excinfo.value), str(excinfo.value)


def test_lists_switch_crc32_blake3_crc64nvme_between_reads(workdir):
    size, shift = 4 * MiB, 16
    path, blake3_text, _ = write_listed_file(workdir, size, shift)
    with open(path, "rb") as f:
        data = f.read()
    texts = {"blake3": blake3_text}
    for algo in ("crc32", "crc64nvme"):
        a = crc_model.ALGOS[algo]
        texts[algo] = "# phase WRITE chunk %d%s\n" % (1 << shift, "" if algo == "crc32" else
                                                      " " + algo) + "".join(
            "%s %d %d %0*x\n" % (path, off, 1 << shift, a.digits,
                                 crc_model.crc(a, data[off:off + (1 << shift)]))
            for off in range(0, size, 1 << shift))
    cfg = WorkerConfig(paths=[path], file_size=size, block_size=MiB, num_threads=2,
                       pipeline_batch_blocks=2)
    with WorkerManager(cfg) as mgr:
        for algo in ("crc32", "blake3", "crc64nvme", "blake3"):
            mgr.set_checksum_list(texts[algo])
            for _ in range(2):  # (the second read replays the graphs the first captured)
                mgr.run_phase(BenchPhase.READFILES)
                assert mgr.checksum_verify_counts() == (size >> shift, 1), algo


def test_infloop_timelimit_read_checks_clean(workdir):
    size, shift = 4 * MiB, 16
    path, text, _ = write_listed_file(workdir, size, shift)
    lst = os.path.join(workdir, "list.txt")
    with open(lst, "w") as f:
        f.write(text)
    res = run_cli("-r", "--infloop", "--timelimit", "2", "-b", "64k", "-s", "4m", "-t", "2",
                  "--rand", "--gpuids", "0", "--nolive", "--checksumverify", lst, path)
    assert res.returncode == 0, res.stderr
    assert "Checksum verify: " in res.stdout


def test_launches_and_copies_match_crc32(workdir):
    path = os.path.join(workdir, "f")
    size, block, shift = 8 * MiB, MiB, 16
    counters = {}
    for name in ("crc32", "blake3"):
        cfg = WorkerConfig(paths=[path], file_size=size, block_size=block, checksums=True,
                           checksum_chunk_shift=shift, checksum_algo=name,
                           pipeline_batch_blocks=2, integrity_check_salt=0xC5C5, staging_engine=2)
        with WorkerManager(cfg) as mgr:
            r = mgr.run_phase(BenchPhase.CREATEFILES)
            counters[name, "write"] = (r["num_kernel_launches"], r["h2d_bytes"], r["d2h_bytes"])
            lines = mgr.checksums()
            if name == "blake3":
                text = list_text(digest_lines(lines), shift)
            else:
                text = "# phase WRITE chunk %d\n" % (1 << shift) + "".join(
                    "%s %d %d %08x\n" % line for line in lines)
            mgr.set_checksum_list(text)
            r = mgr.run_phase(BenchPhase.READFILES)
            counters[name, "read"] = (r["num_kernel_launches"], r["h2d_bytes"], r["d2h_bytes"])
            assert mgr.checksum_verify_counts() == (size >> shift, 1)
    assert counters["crc32", "write"] == counters["blake3", "write"]
    assert counters["crc32", "read"] == counters["blake3", "read"]


def test_cli_whole_file_digest_then_chunked_list(workdir):
    path = os.path.join(workdir, "f")
    sums = os.path.join(workdir, "sums.txt")
    res = run_cli("-w", "-t", "4", "-b", "1m", "-s", "16m", "--blockvarpct", "100", "--gpuids",
                  "0", "--nolive", "--checksums", sums, "--checksumalgo", "blake3", path)
    assert res.returncode == 0, res.stderr
    with open(sums) as f:
        assert f.read() == "# phase WRITE blake3\n%s %d %d %s\n" % (
            path, 16 * MiB, 16 * MiB, file_digest(path, 16 * MiB))
    res = run_cli("-r", "-t", "4", "-b", "1m", "-s", "16m", "--gpuids", "0", "--nolive",
                  "--checksums", sums, "--checksumchunk", "64k", "--checksumalgo", "blake3", path)
    assert res.returncode == 0, res.stderr
    listed = os.path.join(workdir, "list.txt")
    shutil.copy(sums, listed)
    res = run_cli("-r", "--rand", "-t", "4", "-b", "1m", "-s", "16m", "--gpuids", "0", "--nolive",
                  "--checksumverify", listed, path)
    assert res.returncode == 0, res.stderr
    with open(path, "r+b") as f:
        f.seek(5 * MiB + 3)
        f.write(b"\xa5")
    res = run_cli("-r", "-t", "1", "-b", "1m", "-s", "16m", "--gpuids", "0", "--nolive",
                  "--checksumverify", listed, path)
    assert res.returncode != 0
    assert ("Checksum verification failed. File: %s; Offset: %d; Length: 65536; Expected BLAKE3: "
            % (path, 5 * MiB)) in res.stderr + res.stdout
