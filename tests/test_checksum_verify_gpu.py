"""GPU tests of --checksumchunk and --checksumverify: the chunked CRC kernel against zlib for every
chunk of ragged windows, odd addresses and offsets, every length class and one block past 4 GiB;
chunked lists of written data in file, dir and custom tree mode; clean verified reads over the
access patterns, engines and thread counts the list must not depend on; a tree of foreign data;
the error text of a damaged chunk, a missing line and a wrong length; an unchanged clean path; and
the command line."""
import os
import random
import shutil
import zlib

import numpy as np
import pytest
import torch

from tests import test_checksums_gpu as base  # noqa: F401  (sets the mock cuFile library first)
from elbencho_b200 import BenchPhase, WorkerConfig, WorkerError, WorkerManager  # noqa: E402
from elbencho_b200 import kernels  # noqa: E402
from elbencho_b200.worker import IOEngine, PathType  # noqa: E402
from tests.test_checksums_gpu import (CONTENTS, ENGINES, SEED, make_workdir, raw_crc_of,  # noqa: E402
                                      run_cli, setup_mode)

pytestmark = pytest.mark.gpu

KiB, MiB, GiB = 1 << 10, 1 << 20, 1 << 30


# ------------------------------------------------------------------------------------------------
# kernel level
# ------------------------------------------------------------------------------------------------

def chunks_of(offset, length, shift):
    """the chunk indices a block touches"""
    if not length:
        return []
    return list(range(offset >> shift, ((offset + length - 1) >> shift) + 1))


def run_chunks(blocks, shift, slots, shifts=None):
    """blocks: [(device address, length, file offset)] -> the published slots, per block"""
    stream = torch.cuda.current_stream().cuda_stream
    n = len(blocks)
    raw = kernels.pack_block_descs([(ptr, length, off, 0) for ptr, length, off in blocks])
    descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).pin_memory()
    shift_arr = torch.tensor(shifts or [0] * n, dtype=torch.int64).pin_memory()
    dev_crcs = torch.zeros(max(n * slots, 1), dtype=torch.int32, device="cuda")
    host_crcs = torch.full((max(n * slots, 1),), 0x7777, dtype=torch.int32).pin_memory()
    ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
    kernels.crc32_chunks(descs.data_ptr(), shift_arr.data_ptr() if shift == 64 else 0, n, shift,
                         slots, dev_crcs.data_ptr(), host_crcs.data_ptr(), ticket.data_ptr(),
                         stream)
    torch.cuda.synchronize()
    assert int(ticket.item()) == 0 and not dev_crcs.any()
    values = [int(v) & 0xFFFFFFFF for v in host_crcs.tolist()]
    return [values[i * slots:(i + 1) * slots] for i in range(n)]


def expected_chunks(host, base_ptr, blocks, shift, slots):
    """slot j of a block: the raw CRC of its bytes in its (j+1)-th chunk, 0 past its chunks"""
    out = []
    for ptr, length, off in blocks:
        vals = [0] * slots
        for j, c in enumerate(chunks_of(off, length, shift)):
            lo, hi = max(c << shift, off), min((c + 1) << shift, off + length)
            start = ptr - base_ptr + lo - off
            vals[j] = raw_crc_of(host[start:start + hi - lo])
        out.append(vals)
    return out


LENGTHS = [0, 1, 15, 4095, 4 * KiB, MiB]


@pytest.mark.parametrize("shift", [12, 16, 20])
@pytest.mark.parametrize("misalign", [0, 1, 7])
def test_kernel_length_classes(cuda_device, shift, misalign):
    rng = random.Random(shift * 100 + misalign)
    stride = MiB + 8 * KiB
    buf = torch.randint(0, 256, (len(LENGTHS) * stride,), dtype=torch.uint8, device="cuda")
    blocks = []
    for i, length in enumerate(LENGTHS):
        # odd file offsets put chunk boundaries inside a lane's 128 bytes
        off = rng.choice([0, 1 << shift, rng.randrange(1 << 36), (rng.randrange(1 << 30) | 1)])
        blocks.append((buf.data_ptr() + i * stride + misalign, length, off))
    slots = max(len(chunks_of(o, n, shift)) for _, n, o in blocks) + 1
    host = buf.cpu().numpy().tobytes()
    assert run_chunks(blocks, shift, slots) == \
        expected_chunks(host, buf.data_ptr(), blocks, shift, slots)


@pytest.mark.parametrize("seed,num_blocks,max_len,shift", [
    (1, 5, 3 * MiB, 20), (2, 40, 200 * KiB, 16), (3, 300, 9000, 12), (4, 2000, 4 * KiB, 12),
    (5, 64, MiB, 16),
])
def test_kernel_ragged_windows(cuda_device, seed, num_blocks, max_len, shift):
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
    slots = max(len(chunks_of(o, n, shift)) for _, n, o in blocks) or 1
    host = buf.cpu().numpy().tobytes()
    assert run_chunks(blocks, shift, slots) == \
        expected_chunks(host, buf.data_ptr(), blocks, shift, slots)


def test_kernel_full_chunks_finish_to_zlib(cuda_device):
    """the worker's layout: each full chunk's slot finishes to zlib.crc32 of the chunk"""
    shift, length = 16, 4 * MiB
    buf = torch.randint(0, 256, (length,), dtype=torch.uint8, device="cuda")
    (slots,) = run_chunks([(buf.data_ptr(), length, 7 * length)], shift, length >> shift)
    host = buf.cpu().numpy().tobytes()
    for j, raw in enumerate(slots):
        chunk = host[j << shift:(j + 1) << shift]
        assert kernels.crc32_finish(raw, len(chunk)) == zlib.crc32(chunk)


def test_kernel_without_chunks_is_crc32_blocks(cuda_device):
    rng = random.Random(9)
    buf = torch.randint(0, 256, (8 * MiB,), dtype=torch.uint8, device="cuda")
    blocks = [(buf.data_ptr() + rng.randrange(7 * MiB), rng.randrange(MiB), rng.randrange(1 << 40),
               rng.randrange(1 << 40)) for _ in range(50)]
    got = run_chunks([b[:3] for b in blocks], 64, 1, shifts=[b[3] for b in blocks])
    assert [g[0] for g in got] == base.run_kernel(blocks, True)


def test_kernel_block_past_4gib(cuda_device):
    shift, length = 20, 4 * GiB + 4099
    buf = torch.empty(length + 16, dtype=torch.uint8, device="cuda")
    buf.random_(0, 256, generator=torch.Generator("cuda").manual_seed(5))
    ptr = buf.data_ptr() + 5
    num_chunks = (length + (1 << shift) - 1) >> shift
    (slots,) = run_chunks([(ptr, length, 0)], shift, num_chunks)
    host = buf[5:5 + length].cpu().numpy()
    for j in (0, 1, 4095, 4096):
        chunk = host[j << shift:(j + 1) << shift].tobytes()
        assert kernels.crc32_finish(slots[j], len(chunk)) == zlib.crc32(chunk), j
    del buf


def test_kernel_rejects_too_few_slots(cuda_device):
    buf = torch.zeros(64 * KiB, dtype=torch.uint8, device="cuda")
    with pytest.raises(kernels.KernelError, match="spans 2 chunks, more than 1 slots"):
        run_chunks([(buf.data_ptr(), 8 * KiB, 0)], 12, 1)


# ------------------------------------------------------------------------------------------------
# worker level
# ------------------------------------------------------------------------------------------------

@pytest.fixture()
def workdir(cuda_device):
    path = make_workdir()
    yield path
    shutil.rmtree(path, ignore_errors=True)


def list_text(lines, shift, phase="WRITE"):
    return "# phase %s chunk %d\n" % (phase, 1 << shift) + "".join(
        "%s %d %d %08x\n" % line for line in lines)


def check_chunk_lines(lines, files, shift):
    """every chunk of every file once, in order, with zlib.crc32 of its bytes"""
    want = []
    for path in sorted(files):
        with open(path, "rb") as f:
            data = f.read(files[path])
        for off in range(0, files[path], 1 << shift):
            chunk = data[off:off + (1 << shift)]
            want.append((path, off, len(chunk), zlib.crc32(chunk)))
    assert lines == want


WRITE_CONTENTS = {"none": CONTENTS["none"], "blockvar": CONTENTS["blockvar"],
                  "verifyrand": dict(integrity_check_salt=SEED,
                                     integrity_check_kind=kernels.VERIFY_RANDOM)}


@pytest.mark.parametrize("mode,engine,content", [
    (mode, engine, content) for mode in ("file1", "file3", "dir", "tree")
    for engine in ("kernel", "copyengine") for content in WRITE_CONTENTS
    if (mode, content) != ("tree", "verifyrand")])
def test_written_lists_are_zlib_crcs(workdir, mode, engine, content):
    threads = 8 if mode.startswith("file") else 3
    args, files = setup_mode(mode, workdir, threads, False)
    shift = 12 if mode == "tree" else 16
    cfg = WorkerConfig(num_threads=threads, checksums=True, checksum_chunk_shift=shift, **args,
                       **ENGINES[engine], **WRITE_CONTENTS[content])
    with WorkerManager(cfg) as mgr:
        if args.get("path_type") == PathType.DIR:
            mgr.run_phase(BenchPhase.CREATEDIRS)
        mgr.run_phase(BenchPhase.CREATEFILES)
        written = mgr.checksums()
        mgr.set_checksum_list(list_text(written, shift))
        mgr.run_phase(BenchPhase.READFILES)
        read = mgr.checksums()
        counts = mgr.checksum_verify_counts()
    check_chunk_lines(written, files, shift)
    assert read == written
    assert counts == (len(written), len([size for size in files.values() if size]))


def write_listed_file(workdir, size, shift, name="f"):
    path = os.path.join(workdir, name)
    data = np.random.default_rng(size).integers(0, 256, size, dtype=np.uint8).tobytes()
    with open(path, "wb") as f:
        f.write(data)
    lines = [(path, off, len(data[off:off + (1 << shift)]), zlib.crc32(data[off:off + (1 << shift)]))
             for off in range(0, size, 1 << shift)]
    return path, list_text(lines, shift), len(lines)


READS = {
    "seq_b=K": dict(block=1, threads=1),
    "seq_b=4K_8t": dict(block=4, threads=8),
    "rand_b=K_8t": dict(block=1, threads=8, use_random_offsets=True),
    "rand_b=4K_amount": dict(block=4, threads=3, use_random_offsets=True, random_amount=3),
    "aio_qd1": dict(block=1, threads=2, io_engine=IOEngine.AIO, io_depth=1),
    "aio_qd16_rand": dict(block=1, threads=4, io_engine=IOEngine.AIO, io_depth=16,
                          use_random_offsets=True),
    "kernel_staging": dict(block=4, threads=2, staging_engine=1),
    "cufile": dict(block=4, threads=2, use_cufile=True),
}


@pytest.mark.parametrize("shift", [12, 16])
@pytest.mark.parametrize("read", list(READS))
def test_clean_reads_pass(workdir, shift, read):
    opts = dict(READS[read])
    size = 4 * MiB
    path, text, num_lines = write_listed_file(workdir, size, shift)
    block = opts.pop("block") << shift
    threads = opts.pop("threads")
    if "random_amount" in opts:
        opts["random_amount"] *= size
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


def test_clean_direct_read_passes(cuda_device):
    workdir = make_workdir(direct=True)
    try:
        path, text, num_lines = write_listed_file(workdir, 4 * MiB, 16)
        cfg = WorkerConfig(paths=[path], file_size=4 * MiB, block_size=256 * KiB, num_threads=4,
                           use_direct_io=True)
        with WorkerManager(cfg) as mgr:
            mgr.set_checksum_list(text)
            mgr.run_phase(BenchPhase.READFILES)
            assert mgr.checksum_verify_counts() == (num_lines, 1)
    finally:
        shutil.rmtree(workdir, ignore_errors=True)


def test_clean_read_on_two_gpus(workdir):
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    path, text, num_lines = write_listed_file(workdir, 8 * MiB, 16)
    cfg = WorkerConfig(paths=[path], file_size=8 * MiB, block_size=MiB, num_threads=4,
                       gpu_ids=(0, 1))
    with WorkerManager(cfg) as mgr:
        mgr.set_checksum_list(text)
        mgr.run_phase(BenchPhase.READFILES)
        assert mgr.checksum_verify_counts() == (num_lines, 1)


def test_verify_and_checksum_verify_together(workdir):
    path = os.path.join(workdir, "f")
    size, shift = 4 * MiB, 16
    cfg = WorkerConfig(paths=[path], file_size=size, block_size=MiB, num_threads=2, checksums=True,
                       checksum_chunk_shift=shift, integrity_check_salt=SEED,
                       integrity_check_kind=kernels.VERIFY_RANDOM)
    with WorkerManager(cfg) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
        mgr.set_checksum_list(list_text(mgr.checksums(), shift))
        res = mgr.run_phase(BenchPhase.READFILES)
        assert res["verified_bytes"] == size
        assert mgr.checksum_verify_counts() == (size >> shift, 1)


def test_tree_of_foreign_data(workdir):
    """files written outside the tool, read in custom tree mode: a first read lists them, a
    second read verifies against that list"""
    args, files = setup_mode("tree", workdir, 3, False)
    rng = np.random.default_rng(4)
    for path, size in files.items():
        os.makedirs(os.path.dirname(path), exist_ok=True)
        fd = os.open(path, os.O_CREAT | os.O_WRONLY | os.O_TRUNC, 0o644)
        os.write(fd, rng.integers(0, 256, size, dtype=np.uint8).tobytes())
        os.close(fd)
    shift = 12
    with WorkerManager(WorkerConfig(num_threads=3, checksums=True, checksum_chunk_shift=shift,
                                    **args)) as mgr:
        mgr.run_phase(BenchPhase.READFILES)
        listed = mgr.checksums()
    check_chunk_lines(listed, files, shift)
    with WorkerManager(WorkerConfig(num_threads=3, **args)) as mgr:
        mgr.set_checksum_list(list_text(listed, shift, "READ"))
        mgr.run_phase(BenchPhase.READFILES)
        # (an empty file has no chunks)
        assert mgr.checksum_verify_counts() == (len(listed), len([s for s in files.values() if s]))


def failed_read(path, size, text, **kwargs):
    cfg = WorkerConfig(paths=[path], file_size=size, block_size=256 * KiB, num_threads=1,
                       rand_offset_seed=3, **kwargs)
    with WorkerManager(cfg) as mgr:
        mgr.set_checksum_list(text)
        with pytest.raises(WorkerError) as excinfo:
            mgr.run_phase(BenchPhase.READFILES)
    return str(excinfo.value)


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
    msg = failed_read(path, size, text, use_random_offsets=rand)
    assert ("Checksum verification failed. File: %s; Offset: %d; Length: %d; Expected CRC-32: %s; "
            "Actual CRC-32: %08x" % (path, off, 1 << shift, line.rsplit(" ", 1)[1],
                                     zlib.crc32(data[off:off + (1 << shift)]))) in msg, msg


def test_missing_line_and_wrong_length(workdir):
    size, shift = 2 * MiB, 16
    path, text, _ = write_listed_file(workdir, size, shift)
    with open(path, "rb") as f:
        data = f.read()
    lines = text.splitlines(keepends=True)
    missing = "".join(l for l in lines if not l.startswith("%s %d " % (path, MiB)))
    msg = failed_read(path, size, missing)
    assert ("Checksum verification failed. File: %s; Offset: %d; Length: %d; Expected CRC-32: -; "
            "Actual CRC-32: %08x" % (path, MiB, 1 << shift,
                                     zlib.crc32(data[MiB:MiB + (1 << shift)]))) in msg, msg

    wrong = text.replace("%s %d %d " % (path, 0, 1 << shift), "%s %d %d " % (path, 0, 100))
    crc0 = zlib.crc32(data[:1 << shift])
    msg = failed_read(path, size, wrong)
    assert ("Checksum verification failed. File: %s; Offset: 0; Length: %d; Expected CRC-32: "
            "%08x; Actual CRC-32: %08x" % (path, 1 << shift, crc0, crc0)) in msg, msg


def test_clean_path_costs_nothing(workdir):
    """without the options a phase launches and copies what it did before; with
    --checksumverify a read takes one CRC launch per batch more and no copy, and a write none"""
    path = os.path.join(workdir, "f")
    size, block, batch_blocks, shift = 8 * MiB, MiB, 2, 16
    num_batches = size // block // batch_blocks
    counters = {}
    for verify in (False, True):
        cfg = WorkerConfig(paths=[path], file_size=size, block_size=block,
                           pipeline_batch_blocks=batch_blocks, integrity_check_salt=SEED,
                           staging_engine=2)
        with WorkerManager(cfg) as mgr:
            if verify:
                with open(path, "rb") as f:
                    data = f.read()
                mgr.set_checksum_list(list_text(
                    [(path, o, 1 << shift, zlib.crc32(data[o:o + (1 << shift)]))
                     for o in range(0, size, 1 << shift)], shift))
            for phase in (BenchPhase.CREATEFILES, BenchPhase.READFILES):
                r = mgr.run_phase(phase)
                counters[verify, phase] = (r["num_kernel_launches"], r["h2d_bytes"],
                                           r["d2h_bytes"])
    assert counters[False, BenchPhase.CREATEFILES] == (num_batches, 0, size)
    assert counters[False, BenchPhase.READFILES] == (num_batches, size, 0)
    assert counters[True, BenchPhase.CREATEFILES] == (num_batches, 0, size)
    assert counters[True, BenchPhase.READFILES] == (2 * num_batches, size, 0)


# ------------------------------------------------------------------------------------------------
# command line
# ------------------------------------------------------------------------------------------------

def test_cli_write_list_then_verify_random_reads(workdir):
    paths = [os.path.join(workdir, "a"), os.path.join(workdir, "b c")]
    sums = os.path.join(workdir, "sums.txt")
    res = run_cli("-w", "-b", "256k", "-s", "4m", "-t", "4", "--blockvarpct", "100", "--gpuids",
                  "0", "--nolive", "--checksums", sums, "--checksumchunk", "64k", *paths)
    assert res.returncode == 0, res.stderr
    assert "Checksums: 128 chunks in 2 files: %s\n" % sums in res.stdout
    with open(sums) as f:
        text = f.read()
    assert text.startswith("# phase WRITE chunk 65536\n")
    lines = [l.rsplit(" ", 3) for l in text.splitlines()[1:]]
    for path, off, length, crc in lines:
        with open(path, "rb") as f:
            f.seek(int(off))
            assert "%08x" % zlib.crc32(f.read(int(length))) == crc

    res = run_cli("-r", "--rand", "-b", "256k", "-s", "4m", "-t", "4", "--gpuids", "0",
                  "--nolive", "--checksumverify", sums, *paths)
    assert res.returncode == 0, res.stderr
    assert "Checksum verify: 128 chunks checked in 2 files: %s\n" % sums in res.stdout

    res = run_cli("-r", "--infloop", "--timelimit", "2", "-b", "64k", "-s", "4m", "-t", "2",
                  "--gpuids", "0", "--nolive", "--checksumverify", sums, *paths)
    assert res.returncode == 0, res.stderr
    assert "Checksum verify: " in res.stdout

    with open(paths[1], "r+b") as f:
        f.seek(MiB + 5)
        f.write(b"\xff\x00")
    res = run_cli("-r", "-b", "256k", "-s", "4m", "-t", "1", "--gpuids", "0", "--nolive",
                  "--checksumverify", sums, *paths)
    assert res.returncode != 0
    assert "Checksum verification failed. File: %s; Offset: %d; Length: 65536;" % (
        paths[1], MiB) in res.stderr + res.stdout


def test_cli_tree_mode(workdir):
    args, files = setup_mode("tree", workdir, 2, False)
    sums = os.path.join(workdir, "sums.txt")
    common = ["--treefile", args["tree_file_path"], "--treeroundup", "4k", "-b", "64k",
              "--sharesize", "256k", "-t", "2", "--gpuids", "0", "--nolive"]
    res = run_cli("-d", "-w", *common, "--checksums", sums, "--checksumchunk", "4k",
                  args["paths"][0])
    assert res.returncode == 0, res.stderr
    res = run_cli("-r", *common, "--checksumverify", sums, args["paths"][0])
    assert res.returncode == 0, res.stderr
    num_chunks = sum((size + 4095) // 4096 for size in files.values())
    num_files = len([size for size in files.values() if size])
    assert "Checksum verify: %d chunks checked in %d files" % (num_chunks, num_files) in res.stdout


def test_set_checksum_list_rejections(workdir):
    text = "# phase WRITE chunk 65536\n/a 0 65536 00000000\n"
    cases = [
        (dict(checksums=True, checksum_chunk_shift=12),
         "The checksum chunk size (--checksumchunk 4096) differs from the checksum list's (65536)."),
        (dict(block_size=96 * KiB),
         "The block size (98304) is not a multiple of the checksum list's chunk size (65536)."),
        (dict(rwmix_read_percent=10), "Checksum verification (--checksumverify) cannot be used "
         "together with rwmix (a phase in both directions)."),
        (dict(integrity_check_salt=SEED, verify_report=True), "Checksum verification "
         "(--checksumverify) cannot be used together with a verify report (--verifyreport)."),
    ]
    for kwargs, message in cases:
        args = dict(paths=[os.path.join(workdir, "f")], block_size=256 * KiB, file_size=MiB)
        args.update(kwargs)
        with WorkerManager(WorkerConfig(**args)) as mgr:
            with pytest.raises(WorkerError) as excinfo:
                mgr.set_checksum_list(text)
            assert str(excinfo.value) == message
            with pytest.raises(WorkerError, match="^Checksum list line 2: "):
                mgr.set_checksum_list("# phase READ chunk 4096\nbad\n")
