"""Measure --checksums on the GPU (one JSON line per measurement, each with the card's name, power
limit and SM clock limit):

1. the CRC kernel over a 4 GiB resident window of 1 MiB blocks and of 4 KiB blocks, next to the
   verify kernel K2 over the same window and the pinned host-to-device copy rate (CUDA events,
   median of the runs);
2. a 16 GiB file in /dev/shm written and read with 1 MiB blocks and 16 threads, without and with
   --checksums, alternating in one job.

    python scripts/bench_checksums.py [--size-gib 16] [--runs 3] [--dir /dev/shm]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from elbencho_b200 import BenchPhase, WorkerConfig, WorkerManager  # noqa: E402
from elbencho_b200 import kernels  # noqa: E402

KiB, MiB, GiB = 1 << 10, 1 << 20, 1 << 30
SEED = 0xC5C5


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def timed(fn, runs):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    times = []
    for _ in range(runs):
        start.record()
        fn()
        end.record()
        end.synchronize()
        times.append(start.elapsed_time(end) / 1e3)
    return sorted(times)[len(times) // 2]


def descs_of(base, window, block):
    """elb_block_desc[] of a window of equal blocks (file offset = window offset) as a tensor"""
    n = window // block
    arr = np.zeros((n, 4), dtype=np.uint64)
    arr[:, 0] = base + np.arange(n, dtype=np.uint64) * block
    arr[:, 1] = block
    arr[:, 2] = np.arange(n, dtype=np.uint64) * block
    return torch.from_numpy(arr.view(np.uint8).reshape(-1)), n


def kernel_rates(runs, window):
    """GiB/s of the CRC kernel and of K2 per block size, and of a pinned host-to-device copy"""
    stream = torch.cuda.current_stream().cuda_stream
    buf = torch.empty(window, dtype=torch.uint8, device="cuda")
    # the pattern K2 checks, so that it runs its clean path (the CRC does not depend on the bytes)
    kernels.fill_pattern(buf.data_ptr(), window, 0, SEED, stream)
    out = {}

    host = torch.empty(GiB, dtype=torch.uint8).pin_memory()
    dev = buf[:GiB]
    out["pinned H2D copy"] = GiB / GiB / timed(lambda: dev.copy_(host, non_blocking=True), runs)
    del host

    for block in (MiB, 4 * KiB):
        descs, n = descs_of(buf.data_ptr(), window, block)
        pinned_descs = descs.pin_memory()
        dev_descs = descs.cuda()
        shifts = torch.from_numpy((window - np.arange(1, n + 1, dtype=np.uint64) * block)
                                  .astype(np.int64)).pin_memory()
        crcs = torch.zeros(n, dtype=torch.int32, device="cuda")
        host_crcs = torch.zeros(n, dtype=torch.int32).pin_memory()
        ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
        results = torch.empty(n * 2, dtype=torch.int64, device="cuda")
        label = "%d KiB blocks" % (block // KiB)
        out["crc32 " + label] = window / GiB / timed(lambda: kernels.crc32_blocks(
            pinned_descs.data_ptr(), shifts.data_ptr(), n, crcs.data_ptr(), host_crcs.data_ptr(),
            ticket.data_ptr(), stream), runs)
        out["K2 verify_pattern " + label] = window / GiB / timed(
            lambda: kernels.verify_pattern_batch(dev_descs.data_ptr(), n, SEED, results.data_ptr(),
                                                 0, stream, window, block), runs)
    return out


def phase(path, size, bench_phase, checksums):
    cfg = WorkerConfig(paths=[path], block_size=MiB, file_size=size, num_threads=16,
                       checksums=checksums)
    with WorkerManager(cfg) as mgr:
        res = mgr.run_phase(bench_phase)
        lines = mgr.checksums() if checksums else []
    assert not checksums or (len(lines) == 1 and lines[0][3] is not None)
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
    workdir = tempfile.mkdtemp(prefix="elb_bench_checksums_", dir=args.dir)
    path = os.path.join(workdir, "f")
    try:
        for name, bench_phase in (("write", BenchPhase.CREATEFILES),
                                  ("read", BenchPhase.READFILES)):
            for run in range(args.runs):
                for checksums in (False, True):
                    print(json.dumps({"gpu": info, "phase": name, "checksums": checksums,
                                      "run": run, "gib_per_s": phase(path, size, bench_phase,
                                                                     checksums)}), flush=True)
    finally:
        shutil.rmtree(workdir, ignore_errors=True)


if __name__ == "__main__":
    main()
