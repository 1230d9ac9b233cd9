"""Measure --checksumchunk / --checksumverify on the GPU (one JSON line per measurement, each with
the card's name, power limit and SM clock limit):

1. the chunked CRC kernel over a 4 GiB resident window: 1 MiB blocks at K = 4 KiB / 64 KiB /
   1 MiB and 4 KiB blocks at K = 4 KiB, next to the whole-file mode (--checksums), the verify
   kernel K2 over the same window and the pinned host-to-device copy rate (CUDA events, median of
   the runs);
2. reads of a 16 GiB file in /dev/shm with 16 threads, without and with --checksumverify,
   alternating in one job: sequential with 1 MiB blocks at K = 64 KiB, and 4 KiB random reads with
   AIO at queue depth 64 at K = 4 KiB. The lists come from --checksums reads of the same file.

    python scripts/bench_checksum_verify.py [--size-gib 16] [--runs 3] [--dir /dev/shm]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from elbencho_b200 import BenchPhase, WorkerConfig, WorkerManager  # noqa: E402
from elbencho_b200 import kernels  # noqa: E402
from elbencho_b200.worker import IOEngine  # noqa: E402
from scripts.bench_checksums import SEED, descs_of, gpu_info, timed  # noqa: E402

KiB, MiB, GiB = 1 << 10, 1 << 20, 1 << 30


def kernel_rates(runs, window):
    """GiB/s of the chunked and whole-file CRC launches and of K2 per block size, and of a pinned
    host-to-device copy"""
    stream = torch.cuda.current_stream().cuda_stream
    buf = torch.empty(window, dtype=torch.uint8, device="cuda")
    kernels.fill_pattern(buf.data_ptr(), window, 0, SEED, stream)
    out = {}

    host = torch.empty(GiB, dtype=torch.uint8).pin_memory()
    dev = buf[:GiB]
    out["pinned H2D copy"] = 1 / timed(lambda: dev.copy_(host, non_blocking=True), runs)
    del host

    for block, chunk_shifts in ((MiB, (12, 16, 20, 64)), (4 * KiB, (12, 64))):
        descs, n = descs_of(buf.data_ptr(), window, block)
        pinned_descs = descs.pin_memory()
        dev_descs = descs.cuda()
        shifts = torch.from_numpy((window - np.arange(1, n + 1, dtype=np.uint64) * block)
                                  .astype(np.int64)).pin_memory()
        label = "%d KiB blocks" % (block // KiB)
        for shift in chunk_shifts:
            slots = 1 if shift == 64 else block >> shift
            crcs = torch.zeros(n * slots, dtype=torch.int32, device="cuda")
            host_crcs = torch.zeros(n * slots, dtype=torch.int32).pin_memory()
            ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
            name = "crc32 whole file" if shift == 64 else "crc32 chunks K=%d KiB" % (
                (1 << shift) // KiB)
            out["%s, %s" % (name, label)] = window / GiB / timed(lambda: kernels.crc32_chunks(
                pinned_descs.data_ptr(), shifts.data_ptr(), n, shift, slots, crcs.data_ptr(),
                host_crcs.data_ptr(), ticket.data_ptr(), stream), runs)
        results = torch.empty(n * 2, dtype=torch.int64, device="cuda")
        out["K2 verify_pattern, " + label] = window / GiB / timed(
            lambda: kernels.verify_pattern_batch(dev_descs.data_ptr(), n, SEED, results.data_ptr(),
                                                 0, stream, window, block), runs)
    return out


READS = {
    "seq 1 MiB, K=64 KiB": (16, dict(block_size=MiB)),
    "rand 4 KiB qd64, K=4 KiB": (12, dict(block_size=4 * KiB, use_random_offsets=True,
                                          io_engine=IOEngine.AIO, io_depth=64, rand_offset_seed=7)),
}


def read_rate(path, size, shift, opts, checksum_list, random_amount):
    cfg = WorkerConfig(paths=[path], file_size=size, num_threads=16,
                       random_amount=random_amount if opts.get("use_random_offsets") else 0,
                       **opts)
    with WorkerManager(cfg) as mgr:
        if checksum_list:
            mgr.set_checksum_list(checksum_list)
        res = mgr.run_phase(BenchPhase.READFILES)
        if checksum_list:
            chunks, _ = mgr.checksum_verify_counts()
            assert chunks == res["ops_total"]["bytes"] >> shift
    return round(res["ops_total"]["bytes"] / GiB / (res["last_finish_usec"] / 1e6), 3)


def make_list(path, size, shift):
    cfg = WorkerConfig(paths=[path], file_size=size, block_size=MiB, num_threads=16,
                       checksums=True, checksum_chunk_shift=shift)
    with WorkerManager(cfg) as mgr:
        mgr.run_phase(BenchPhase.READFILES)
        return "# phase READ chunk %d\n" % (1 << shift) + mgr.checksums_text()


def main():
    parser = argparse.ArgumentParser()
    parser.add_argument("--size-gib", type=int, default=16)
    parser.add_argument("--window-gib", type=int, default=4)
    parser.add_argument("--rand-gib", type=int, default=4, help="bytes of each random read")
    parser.add_argument("--runs", type=int, default=3)
    parser.add_argument("--dir", default="/dev/shm")
    args = parser.parse_args()
    torch.cuda.set_device(0)
    info = gpu_info()

    for name, rate in kernel_rates(max(args.runs, 5), args.window_gib * GiB).items():
        print(json.dumps({"gpu": info, "kernel": name, "window_gib": args.window_gib,
                          "gib_per_s": round(rate, 1)}), flush=True)
    torch.cuda.empty_cache()

    size = args.size_gib * GiB
    workdir = tempfile.mkdtemp(prefix="elb_bench_checksum_verify_", dir=args.dir)
    path = os.path.join(workdir, "f")
    try:
        with WorkerManager(WorkerConfig(paths=[path], block_size=MiB, file_size=size,
                                        num_threads=16, block_variance_percent=100)) as mgr:
            mgr.run_phase(BenchPhase.CREATEFILES)
        for name, (shift, opts) in READS.items():
            checksum_list = make_list(path, size, shift)
            for run in range(args.runs):
                for verify in (False, True):
                    rate = read_rate(path, size, shift, opts, checksum_list if verify else None,
                                     args.rand_gib * GiB)
                    print(json.dumps({"gpu": info, "read": name, "checksumverify": verify,
                                      "run": run, "gib_per_s": rate}), flush=True)
    finally:
        shutil.rmtree(workdir, ignore_errors=True)


if __name__ == "__main__":
    main()
