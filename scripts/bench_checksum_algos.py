"""Measure --checksumalgo on the GPU (one JSON line per measurement, each with the card's name, power
limit and SM clock limit):

1. the pinned host-to-device copy rate, and the checksum kernel of each algorithm (crc32, crc32c,
   crc64nvme, blake3) over a 4 GiB resident window of 1 MiB and of 4 KiB blocks at K = 4 KiB /
   64 KiB / 1 MiB (1 MiB blocks only) and whole files (CUDA events, median of the runs);
2. sequential 1 MiB reads of a 16 GiB file in /dev/shm with 16 threads and --checksumverify at
   K = 64 KiB, against a crc32, a crc64nvme and a blake3 list of the file, alternating in one job;
3. sequential 4 KiB reads of the same file with 16 threads, without checksums and with whole-file
   blake3 --checksums, alternating: the cost of the host merge of the BLAKE3 runs.

    python scripts/bench_checksum_algos.py [--size-gib 16] [--runs 3] [--dir /dev/shm]
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
from scripts.bench_checksums import SEED, descs_of, gpu_info, timed  # noqa: E402

KiB, MiB, GiB = 1 << 10, 1 << 20, 1 << 30
ALGOS = ("crc32", "crc32c", "crc64nvme", "blake3")


def kernel_rates(runs, window):
    """GiB/s of the pinned host-to-device copy and of each algorithm's CRC launch per block size
    and chunk size"""
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
        shifts = torch.from_numpy((window - np.arange(1, n + 1, dtype=np.uint64) * block)
                                  .astype(np.int64)).pin_memory()
        label = "%d KiB blocks" % (block // KiB)
        for shift in chunk_shifts:
            slots = 1 if shift == 64 else block >> shift
            chunk = "whole file" if shift == 64 else "K=%d KiB" % ((1 << shift) // KiB)
            for algo in ALGOS:
                if algo == "blake3":
                    # whole files: a slot per run, 2 log2(chunks per block) + 1 at most
                    b3_slots = (2 * ((block // KiB).bit_length() - 1) + 1) if shift == 64 else slots
                    digests = torch.zeros(n * b3_slots * 32, dtype=torch.uint8, device="cuda")
                    host_digests = torch.zeros(n * b3_slots * 32, dtype=torch.uint8).pin_memory()
                    ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
                    out["%s %s, %s" % (algo, chunk, label)] = window / GiB / timed(
                        lambda: kernels.blake3_chunks(pinned_descs.data_ptr(), shifts.data_ptr(),
                                                      n, shift, b3_slots, digests.data_ptr(),
                                                      host_digests.data_ptr(), ticket.data_ptr(),
                                                      stream), runs)
                    del digests, host_digests
                    continue
                dtype = torch.int64 if algo == "crc64nvme" else torch.int32
                crcs = torch.zeros(n * slots, dtype=dtype, device="cuda")
                host_crcs = torch.zeros(n * slots, dtype=dtype).pin_memory()
                ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
                out["%s %s, %s" % (algo, chunk, label)] = window / GiB / timed(
                    lambda: kernels.crc_chunks(pinned_descs.data_ptr(), shifts.data_ptr(), n,
                                               shift, slots, crcs.data_ptr(),
                                               host_crcs.data_ptr(), ticket.data_ptr(), stream,
                                               algo=algo), runs)
                del crcs, host_crcs
    return out


def read_rate(path, size, checksum_list):
    cfg = WorkerConfig(paths=[path], file_size=size, num_threads=16, block_size=MiB)
    with WorkerManager(cfg) as mgr:
        mgr.set_checksum_list(checksum_list)
        res = mgr.run_phase(BenchPhase.READFILES)
        chunks, _ = mgr.checksum_verify_counts()
        assert chunks == size >> 16
    return round(res["ops_total"]["bytes"] / GiB / (res["last_finish_usec"] / 1e6), 3)


def make_list(path, size, algo):
    cfg = WorkerConfig(paths=[path], file_size=size, block_size=MiB, num_threads=16,
                       checksums=True, checksum_chunk_shift=16, checksum_algo=algo)
    with WorkerManager(cfg) as mgr:
        mgr.run_phase(BenchPhase.READFILES)
        return ("# phase READ chunk 65536%s\n" % ("" if algo == "crc32" else " " + algo) +
                mgr.checksums_text())


def whole_file_read_rate(path, size, checksums):
    cfg = WorkerConfig(paths=[path], file_size=size, num_threads=16, block_size=4 * KiB,
                       checksums=checksums, checksum_algo="blake3")
    with WorkerManager(cfg) as mgr:
        res = mgr.run_phase(BenchPhase.READFILES)
        if checksums:
            ((_, _, covered, digest),) = mgr.checksums()
            assert covered == size and digest is not None
    return round(res["ops_total"]["bytes"] / GiB / (res["last_finish_usec"] / 1e6), 3)


def main():
    parser = argparse.ArgumentParser()
    parser.add_argument("--size-gib", type=int, default=16)
    parser.add_argument("--window-gib", type=int, default=4)
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
    workdir = tempfile.mkdtemp(prefix="elb_bench_checksum_algos_", dir=args.dir)
    path = os.path.join(workdir, "f")
    try:
        with WorkerManager(WorkerConfig(paths=[path], block_size=MiB, file_size=size,
                                        num_threads=16, block_variance_percent=100)) as mgr:
            mgr.run_phase(BenchPhase.CREATEFILES)
        lists = {algo: make_list(path, size, algo) for algo in ("crc32", "crc64nvme", "blake3")}
        for run in range(args.runs):
            for algo in ("crc32", "crc64nvme", "blake3"):
                rate = read_rate(path, size, lists[algo])
                print(json.dumps({"gpu": info, "read": "seq 1 MiB, K=64 KiB, --checksumverify",
                                  "algo": algo, "run": run, "gib_per_s": rate}), flush=True)
        for run in range(args.runs):
            for checksums in (False, True):
                rate = whole_file_read_rate(path, size, checksums)
                print(json.dumps({"gpu": info, "read": "seq 4 KiB, whole file",
                                  "checksums": "blake3" if checksums else "none", "run": run,
                                  "gib_per_s": rate}), flush=True)
    finally:
        shutil.rmtree(workdir, ignore_errors=True)


if __name__ == "__main__":
    main()
