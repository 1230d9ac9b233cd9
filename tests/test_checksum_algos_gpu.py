"""GPU tests of --checksumalgo, each for CRC-32, CRC-32C and CRC-64/NVME: the CRC kernel against the
model (tests/crc_algo_model.py) at chunks of 4 KiB, 64 KiB, 1 MiB and whole files, for odd addresses
and offsets, every length class, ragged windows, a block past 4 GiB and whole-file shifts past 2^31,
2^32 and near 2^64; written lists in file, dir and custom tree mode; clean verified reads over the
access patterns and engines; the error text of a damaged chunk; a list of another algorithm between
two read phases; the launches and copies of a run; and the command line."""
import functools
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
from tests import crc_algo_model as model  # noqa: E402
from tests.test_checksums_gpu import (SEED, make_workdir, run_cli, setup_mode)  # noqa: E402

pytestmark = pytest.mark.gpu

KiB, MiB, GiB = 1 << 10, 1 << 20, 1 << 30
ALGOS = list(model.ALGOS)
PIECE = 4 * KiB


# ------------------------------------------------------------------------------------------------
# the model at the sizes of these tests: the model's byte table over many 4 KiB pieces at once,
# joined by the model's X
# ------------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def _table(name):
    a = model.ALGOS[name]
    return np.array([model.raw_crc(a, bytes([i])) for i in range(256)], dtype=np.uint64)


@functools.lru_cache(maxsize=None)
def _x8n(name, n):
    a = model.ALGOS[name]
    return model._xpow(a, 8 * n)


def _join(name, crc, n, tail_crc):
    """R(A || B) from crc = R(A), n = |B| and tail_crc = R(B)"""
    a = model.ALGOS[name]
    shifted = model._reflect(a, model._polymulmod(a, model._reflect(a, crc), _x8n(name, n)))
    return shifted ^ tail_crc


def raw_crc(name, data):
    """R(data): the pieces' Rs side by side (zeros in front of a piece do not change its R)"""
    data = bytes(data)
    table = _table(name)
    if len(data) <= PIECE:
        crc = 0
        for byte in data:
            crc = int(table[(crc ^ byte) & 0xFF]) ^ (crc >> 8)
        return crc
    num = (len(data) + PIECE - 1) // PIECE
    pad = num * PIECE - len(data)
    arr = np.frombuffer(bytes(pad) + data, dtype=np.uint8).reshape(num, PIECE)
    crcs = np.zeros(num, dtype=np.uint64)
    for i in range(PIECE):
        crcs = table[(crcs ^ arr[:, i]) & np.uint64(0xFF)] ^ (crcs >> np.uint64(8))
    crc = 0
    for piece_crc in crcs.tolist():
        crc = _join(name, crc, PIECE, int(piece_crc))
    return crc


def published_crc(name, data):
    return model.finish(model.ALGOS[name], raw_crc(name, data), len(data))


# ------------------------------------------------------------------------------------------------
# kernel level
# ------------------------------------------------------------------------------------------------

def chunks_of(offset, length, shift):
    if not length:
        return []
    if shift == 64:
        return [0]
    return list(range(offset >> shift, ((offset + length - 1) >> shift) + 1))


def run_chunks(name, blocks, shift, slots, shifts=None):
    """blocks: [(device address, length, file offset)] -> the published slots, per block"""
    a = model.ALGOS[name]
    dtype = torch.int64 if a.width == 64 else torch.int32
    stream = torch.cuda.current_stream().cuda_stream
    n = len(blocks)
    raw = kernels.pack_block_descs([(ptr, length, off, 0) for ptr, length, off in blocks])
    descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).pin_memory()
    shift_arr = torch.tensor([s - (1 << 64) if s >> 63 else s for s in (shifts or [0] * n)],
                             dtype=torch.int64).pin_memory()
    dev_crcs = torch.zeros(max(n * slots, 1), dtype=dtype, device="cuda")
    host_crcs = torch.full((max(n * slots, 1),), 0x7777, dtype=dtype).pin_memory()
    ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
    before = kernels.num_kernel_launches()
    kernels.crc_chunks(descs.data_ptr(), shift_arr.data_ptr() if shift == 64 else 0, n, shift,
                       slots, dev_crcs.data_ptr(), host_crcs.data_ptr(), ticket.data_ptr(), stream,
                       algo=name)
    torch.cuda.synchronize()
    assert kernels.num_kernel_launches() == before + (1 if n else 0)
    assert int(ticket.item()) == 0 and not dev_crcs.any()
    values = [int(v) & a.mask for v in host_crcs.tolist()]
    return [values[i * slots:(i + 1) * slots] for i in range(n)]


def expected_chunks(name, host, base_ptr, blocks, shift, slots, shifts=None):
    """slot j of a block: the raw CRC of its bytes in its (j+1)-th chunk (whole files: shifted by
    the block's shift), 0 past its chunks"""
    a = model.ALGOS[name]
    out = []
    for i, (ptr, length, off) in enumerate(blocks):
        vals = [0] * slots
        for j, c in enumerate(chunks_of(off, length, shift)):
            lo, hi = (off, off + length) if shift == 64 else \
                (max(c << shift, off), min((c + 1) << shift, off + length))
            start = ptr - base_ptr + lo - off
            vals[j] = raw_crc(name, host[start:start + hi - lo])
            if shift == 64:
                vals[j] = model.shift(a, vals[j], shifts[i])
        out.append(vals)
    return out


LENGTHS = [0, 1, 15, 4095, 4 * KiB, 4 * KiB + 1, MiB + 13]


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("shift", [12, 16, 20, 64])
@pytest.mark.parametrize("misalign", [0, 1, 7])
def test_kernel_length_classes(cuda_device, algo, shift, misalign):
    rng = random.Random(shift * 100 + misalign)
    stride = MiB + 8 * KiB
    buf = torch.randint(0, 256, (len(LENGTHS) * stride,), dtype=torch.uint8, device="cuda")
    blocks = []
    for i, length in enumerate(LENGTHS):
        # odd file offsets put chunk boundaries inside a lane's 128 bytes
        off = rng.choice([0, 1 << min(shift, 40), rng.randrange(1 << 36),
                          (rng.randrange(1 << 30) | 1)])
        blocks.append((buf.data_ptr() + i * stride + misalign, length, off))
    shifts = [rng.randrange(1 << 40) for _ in blocks]
    slots = 1 if shift == 64 else max(len(chunks_of(o, n, shift)) for _, n, o in blocks) + 1
    host = buf.cpu().numpy().tobytes()
    assert run_chunks(algo, blocks, shift, slots, shifts) == \
        expected_chunks(algo, host, buf.data_ptr(), blocks, shift, slots, shifts)


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("seed,num_blocks,max_len,shift", [
    (1, 5, 3 * MiB, 20), (2, 40, 200 * KiB, 16), (3, 300, 9000, 12), (4, 1000, 4 * KiB, 12),
    (5, 64, 256 * KiB, 64),
])
def test_kernel_ragged_windows(cuda_device, algo, seed, num_blocks, max_len, shift):
    rng = random.Random(seed)
    slot_bytes = max_len + 32
    buf = torch.randint(0, 256, (num_blocks * slot_bytes,), dtype=torch.uint8, device="cuda",
                        generator=torch.Generator("cuda").manual_seed(seed))
    blocks = []
    for i in range(num_blocks):
        length = rng.choice([0, 1, rng.randint(0, max_len), max_len])
        # half the blocks in the worker's layout (address = offset mod 4 KiB), half anywhere
        off = rng.randrange(1 << 34)
        ptr = buf.data_ptr() + i * slot_bytes + rng.randrange(16)
        if i % 2:
            off = (off & ~4095) | (ptr & 4095)
        blocks.append((ptr, length, off))
    shifts = [rng.randrange(1 << 34) for _ in blocks]
    slots = max(len(chunks_of(o, n, shift)) for _, n, o in blocks) or 1
    host = buf.cpu().numpy().tobytes()
    assert run_chunks(algo, blocks, shift, slots, shifts) == \
        expected_chunks(algo, host, buf.data_ptr(), blocks, shift, slots, shifts)


@pytest.mark.parametrize("algo", ALGOS)
def test_kernel_whole_file_shifts_past_2g_4g_and_near_2_64(cuda_device, algo):
    """shifts given directly: the shift chain's reduction by the algorithm's order of x"""
    buf = torch.randint(0, 256, (64 * KiB,), dtype=torch.uint8, device="cuda",
                        generator=torch.Generator("cuda").manual_seed(11))
    shifts = [(1 << 31) - 1, 1 << 31, (1 << 31) + 4096, (1 << 32) - 1, 1 << 32, (1 << 32) + 77,
              5 << 32, (1 << 62) + 3, (1 << 64) - 4096, (1 << 64) - 2, (1 << 64) - 1]
    blocks = [(buf.data_ptr() + 3 * i, 5000 + 4096 * (i % 3), 0) for i in range(len(shifts))]
    host = buf.cpu().numpy().tobytes()
    assert run_chunks(algo, blocks, 64, 1, shifts) == \
        expected_chunks(algo, host, buf.data_ptr(), blocks, 64, 1, shifts)


@pytest.mark.parametrize("algo", ALGOS)
def test_kernel_full_chunks_finish_to_the_published_crc(cuda_device, algo):
    shift, length = 16, 2 * MiB
    buf = torch.randint(0, 256, (length,), dtype=torch.uint8, device="cuda")
    (slots,) = run_chunks(algo, [(buf.data_ptr(), length, 7 * length)], shift, length >> shift)
    host = buf.cpu().numpy().tobytes()
    for j, raw in enumerate(slots):
        chunk = host[j << shift:(j + 1) << shift]
        assert kernels.crc_finish(raw, len(chunk), algo=algo) == published_crc(algo, chunk)


@pytest.mark.parametrize("algo", ALGOS)
def test_kernel_block_past_4gib(cuda_device, algo):
    shift, length = 20, 4 * GiB + 4099
    buf = torch.empty(length + 16, dtype=torch.uint8, device="cuda")
    buf.random_(0, 256, generator=torch.Generator("cuda").manual_seed(5))
    ptr = buf.data_ptr() + 5
    num_chunks = (length + (1 << shift) - 1) >> shift
    (slots,) = run_chunks(algo, [(ptr, length, 0)], shift, num_chunks)
    for j in (0, 1, 4095, 4096):
        chunk = buf[5 + (j << shift):5 + min((j + 1) << shift, length)].cpu().numpy().tobytes()
        assert kernels.crc_finish(slots[j], len(chunk), algo=algo) == \
            published_crc(algo, chunk), j
    del buf
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------
# worker level
# ------------------------------------------------------------------------------------------------

@pytest.fixture()
def workdir(cuda_device):
    path = make_workdir()
    yield path
    shutil.rmtree(path, ignore_errors=True)


def header(name, shift=None, phase="WRITE"):
    return "# phase %s%s%s\n" % (phase, "" if shift is None else " chunk %d" % (1 << shift),
                                 "" if name == "crc32" else " " + name)


def list_text(name, lines, shift, phase="WRITE"):
    digits = model.ALGOS[name].digits
    return header(name, shift, phase) + "".join(
        "%s %d %d %0*x\n" % (path, off, length, digits, crc) for path, off, length, crc in lines)


def file_chunks(name, files, shift):
    """every chunk of every file once, in order, with its CRC"""
    want = []
    for path in sorted(files):
        with open(path, "rb") as f:
            data = f.read(files[path])
        for off in range(0, files[path], 1 << shift):
            chunk = data[off:off + (1 << shift)]
            want.append((path, off, len(chunk), published_crc(name, chunk)))
    return want


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("mode", ["file1", "file3", "dir", "tree"])
def test_written_lists_match_the_model(workdir, algo, mode):
    threads = 4 if mode.startswith("file") else 3
    args, files = setup_mode(mode, workdir, threads, False)
    shift = 12 if mode == "tree" else 16
    content = {} if mode == "tree" else dict(block_variance_percent=100)
    cfg = WorkerConfig(num_threads=threads, checksums=True, checksum_chunk_shift=shift,
                       checksum_algo=algo, **args, **content)
    with WorkerManager(cfg) as mgr:
        if args.get("path_type") == PathType.DIR:
            mgr.run_phase(BenchPhase.CREATEDIRS)
        mgr.run_phase(BenchPhase.CREATEFILES)
        written = mgr.checksums()
        mgr.set_checksum_list(list_text(algo, written, shift))
        mgr.run_phase(BenchPhase.READFILES)
        read = mgr.checksums()
        counts = mgr.checksum_verify_counts()
    assert written == file_chunks(algo, files, shift)
    assert read == written
    assert counts == (len(written), len([size for size in files.values() if size]))
    # whole files: one line per file with the CRC of all its bytes
    cfg = WorkerConfig(num_threads=threads, checksums=True, checksum_algo=algo, **args)
    with WorkerManager(cfg) as mgr:
        mgr.run_phase(BenchPhase.READFILES)
        lines = mgr.checksums()
    want = []
    for path in sorted(files):
        with open(path, "rb") as f:
            want.append((path, files[path], files[path], published_crc(algo, f.read())))
    assert lines == want


def write_listed_file(name, workdir, size, shift, fname="f"):
    path = os.path.join(workdir, fname)
    data = np.random.default_rng(size).integers(0, 256, size, dtype=np.uint8).tobytes()
    with open(path, "wb") as f:
        f.write(data)
    lines = file_chunks(name, {path: size}, shift)
    return path, list_text(name, lines, shift), len(lines)


READS = {
    "seq": dict(block=4, threads=2),
    "rand": dict(block=1, threads=4, use_random_offsets=True),
    "sync_qd1": dict(block=4, threads=2, io_engine=IOEngine.SYNC),
    "aio_qd16": dict(block=1, threads=4, io_engine=IOEngine.AIO, io_depth=16),
    "aio_qd16_rand": dict(block=1, threads=4, io_engine=IOEngine.AIO, io_depth=16,
                          use_random_offsets=True),
    "kernel_staging": dict(block=4, threads=2, staging_engine=1),
    "cufile": dict(block=4, threads=2, use_cufile=True),
}


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("read", list(READS))
def test_clean_reads_pass(workdir, algo, read):
    opts = dict(READS[read])
    size, shift = 4 * MiB, 16
    path, text, num_lines = write_listed_file(algo, workdir, size, shift)
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


@pytest.mark.parametrize("algo", ALGOS)
def test_clean_direct_read_passes(cuda_device, algo):
    workdir = make_workdir(direct=True)
    try:
        path, text, num_lines = write_listed_file(algo, workdir, 4 * MiB, 16)
        cfg = WorkerConfig(paths=[path], file_size=4 * MiB, block_size=256 * KiB, num_threads=4,
                           use_direct_io=True)
        with WorkerManager(cfg) as mgr:
            mgr.set_checksum_list(text)
            mgr.run_phase(BenchPhase.READFILES)
            assert mgr.checksum_verify_counts() == (num_lines, 1)
    finally:
        shutil.rmtree(workdir, ignore_errors=True)


LABELS = {"crc32": "CRC-32", "crc32c": "CRC-32C", "crc64nvme": "CRC-64/NVME"}


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("rand", [False, True])
def test_flipped_byte_names_its_chunk(workdir, algo, rand):
    size, shift = 4 * MiB, 16
    path, text, _ = write_listed_file(algo, workdir, size, shift)
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
    label, digits = LABELS[algo], model.ALGOS[algo].digits
    assert ("Checksum verification failed. File: %s; Offset: %d; Length: %d; Expected %s: %s; "
            "Actual %s: %0*x" % (path, off, 1 << shift, label, line.rsplit(" ", 1)[1], label,
                                 digits, published_crc(algo, data[off:off + (1 << shift)]))
            ) in str(excinfo.value), str(excinfo.value)


def test_list_of_another_algorithm_between_read_phases(workdir):
    """each list's algorithm re-makes the slots and the batch graphs: every read checks with the
    list it was given, and a wrong line of the last list fails with that list's algorithm"""
    size, shift = 4 * MiB, 16
    path = os.path.join(workdir, "f")
    texts = {}
    with open(path, "wb") as f:
        f.write(np.random.default_rng(8).integers(0, 256, size, dtype=np.uint8).tobytes())
    for algo in ("crc32c", "crc64nvme", "crc32"):
        texts[algo] = list_text(algo, file_chunks(algo, {path: size}, shift), shift)
    cfg = WorkerConfig(paths=[path], file_size=size, block_size=MiB, num_threads=2,
                       pipeline_batch_blocks=2)
    with WorkerManager(cfg) as mgr:
        for algo in ("crc32c", "crc64nvme", "crc32", "crc64nvme", "crc32c"):
            mgr.set_checksum_list(texts[algo])
            for _ in range(2):  # (the second read replays the graphs the first captured)
                mgr.run_phase(BenchPhase.READFILES)
                assert mgr.checksum_verify_counts() == (size >> shift, 1), algo
        lines = texts["crc64nvme"].splitlines(keepends=True)
        crc = int(lines[5].rsplit(" ", 1)[1], 16)
        lines[5] = lines[5].rsplit(" ", 1)[0] + " %016x\n" % (crc ^ (1 << 63))
        mgr.set_checksum_list("".join(lines))
        with pytest.raises(WorkerError, match="Expected CRC-64/NVME: %016x; Actual CRC-64/NVME: "
                           "%016x" % (crc ^ (1 << 63), crc)):
            mgr.run_phase(BenchPhase.READFILES)


def test_configured_algorithm_must_match_the_list(workdir):
    text = "# phase WRITE chunk 65536 crc32c\n/a 0 65536 00000000\n"
    cfg = WorkerConfig(paths=[os.path.join(workdir, "f")], block_size=256 * KiB, file_size=MiB,
                       checksums=True, checksum_algo="crc64nvme")
    with WorkerManager(cfg) as mgr:
        with pytest.raises(WorkerError) as excinfo:
            mgr.set_checksum_list(text)
        assert str(excinfo.value) == ("The checksum algorithm (--checksumalgo crc64nvme) differs "
                                      "from the checksum list's (crc32c).")
        mgr.set_checksum_list(text.replace("crc32c\n/a 0 65536 00000000",
                                           "crc64nvme\n/a 0 65536 0000000000000000"))


@pytest.mark.parametrize("algo", ["crc32c", "crc64nvme"])
def test_launches_and_copies_match_crc32(workdir, algo):
    """a run of another algorithm launches and copies what a crc32 run does, in a write phase
    with --checksums and a read phase with a list"""
    path = os.path.join(workdir, "f")
    size, block, shift = 8 * MiB, MiB, 16
    counters = {}
    for name in ("crc32", algo):
        cfg = WorkerConfig(paths=[path], file_size=size, block_size=block, checksums=True,
                           checksum_chunk_shift=shift, checksum_algo=name,
                           pipeline_batch_blocks=2, integrity_check_salt=SEED, staging_engine=2)
        with WorkerManager(cfg) as mgr:
            r = mgr.run_phase(BenchPhase.CREATEFILES)
            counters[name, "write"] = (r["num_kernel_launches"], r["h2d_bytes"], r["d2h_bytes"])
            mgr.set_checksum_list(list_text(name, mgr.checksums(), shift))
            r = mgr.run_phase(BenchPhase.READFILES)
            counters[name, "read"] = (r["num_kernel_launches"], r["h2d_bytes"], r["d2h_bytes"])
            assert mgr.checksum_verify_counts() == (size >> shift, 1)
    num_batches = size // block // 2
    assert counters["crc32", "write"] == counters[algo, "write"] == (2 * num_batches, 0, size)
    assert counters["crc32", "read"] == counters[algo, "read"] == (2 * num_batches, size, 0)


# ------------------------------------------------------------------------------------------------
# command line
# ------------------------------------------------------------------------------------------------

def test_cli_write_crc64nvme_list_then_verify_random_reads(workdir):
    paths = [os.path.join(workdir, "a"), os.path.join(workdir, "b c")]
    sums = os.path.join(workdir, "sums.txt")
    res = run_cli("-w", "-b", "256k", "-s", "4m", "-t", "4", "--blockvarpct", "100", "--gpuids",
                  "0", "--nolive", "--checksums", sums, "--checksumchunk", "64k",
                  "--checksumalgo", "crc64nvme", *paths)
    assert res.returncode == 0, res.stderr
    assert "Checksums: 128 chunks in 2 files: %s\n" % sums in res.stdout
    with open(sums) as f:
        text = f.read()
    assert text.startswith("# phase WRITE chunk 65536 crc64nvme\n")
    for line in text.splitlines()[1:]:
        path, off, length, crc = line.rsplit(" ", 3)
        with open(path, "rb") as f:
            f.seek(int(off))
            assert "%016x" % published_crc("crc64nvme", f.read(int(length))) == crc

    res = run_cli("-r", "--rand", "-b", "256k", "-s", "4m", "-t", "4", "--gpuids", "0",
                  "--nolive", "--checksumverify", sums, *paths)
    assert res.returncode == 0, res.stderr
    assert "Checksum verify: 128 chunks checked in 2 files: %s\n" % sums in res.stdout

    with open(paths[1], "r+b") as f:
        f.seek(MiB + 5)
        f.write(b"\xff\x00")
    res = run_cli("-r", "-b", "256k", "-s", "4m", "-t", "1", "--gpuids", "0", "--nolive",
                  "--checksumverify", sums, *paths)
    assert res.returncode != 0
    assert ("Checksum verification failed. File: %s; Offset: %d; Length: 65536; Expected "
            "CRC-64/NVME: " % (paths[1], MiB)) in res.stderr + res.stdout


@pytest.mark.parametrize("algo", ["crc32c", "crc64nvme"])
def test_cli_whole_file_section(workdir, algo):
    path = os.path.join(workdir, "f")
    sums = os.path.join(workdir, "sums.txt")
    res = run_cli("-w", "-r", "-b", "1m", "-s", "3m", "--blockvarpct", "100", "--gpuids", "0",
                  "--nolive", "--checksums", sums, "--checksumalgo", algo, path)
    assert res.returncode == 0, res.stderr
    with open(path, "rb") as f:
        want = "%s %d %d %0*x\n" % (path, 3 * MiB, 3 * MiB, model.ALGOS[algo].digits,
                                    published_crc(algo, f.read()))
    with open(sums) as f:
        assert f.read() == header(algo) + want + header(algo, phase="READ") + want
