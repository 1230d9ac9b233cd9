"""Measure --verifyreport on the GPU (one JSON line per measurement):

1. the damage map kernel over a fully damaged 1 GiB resident window of 1 MiB blocks, next to the
   verify kernels K2 / K4 / K6 over the same window (CUDA events, median of the runs);
2. a 16 GiB file in /dev/shm read with 1 MiB blocks and 16 threads: clean without and with the
   report (alternating), then with 1 % of the blocks damaged and with every block damaged (read
   with another seed), with the report.

    python scripts/bench_verify_report.py [--size-gib 16] [--runs 3] [--dir /dev/shm]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

from elbencho_b200 import BenchPhase, WorkerConfig, WorkerError, WorkerManager  # noqa: E402
from elbencho_b200 import kernels  # noqa: E402

MiB, GiB = 1 << 20, 1 << 30
SEED = 0xBE7C


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


def kernel_rates(runs):
    """GiB/s of K2 / K4 / K6 and of the damage map over a 1 GiB window of 1 MiB blocks"""
    stream = torch.cuda.current_stream().cuda_stream
    n = 1024
    buf = torch.empty(n * MiB, dtype=torch.uint8, device="cuda")
    blocks = [(buf.data_ptr() + i * MiB, MiB, i * MiB, i) for i in range(n)]
    descs = torch.frombuffer(bytearray(kernels.pack_block_descs(blocks)), dtype=torch.uint8)
    dev_descs = descs.cuda()
    pinned_descs = descs.pin_memory()
    results = torch.empty(n * 2, dtype=torch.int64, device="cuda")
    per_desc = MiB // 512
    sectors = torch.empty(n * per_desc * 4, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    out = {}
    ops = {
        "K2 verify_pattern": lambda: kernels.verify_pattern_batch(
            dev_descs.data_ptr(), n, SEED, results.data_ptr(), 0, stream, n * MiB, MiB),
        "K4 verify_random": lambda: kernels.verify_random_batch(
            dev_descs.data_ptr(), n, 100, SEED, results.data_ptr(), 0, stream, n * MiB, MiB),
        "K6 verify_random_grain": lambda: kernels.verify_random_grain_batch(
            dev_descs.data_ptr(), n, 16, 100, SEED, results.data_ptr(), 0, stream, n * MiB, MiB),
        "damage_map random_grain": lambda: kernels.damage_map(
            pinned_descs.data_ptr(), n, kernels.CONTENT_RANDOM_GRAIN, SEED, 100, 16, 0,
            sectors.data_ptr(), per_desc, stream),
        "damage_map pattern": lambda: kernels.damage_map(
            pinned_descs.data_ptr(), n, kernels.CONTENT_PATTERN, SEED, 0, 0, 0,
            sectors.data_ptr(), per_desc, stream),
    }
    # the window holds random bytes: every block and almost every byte differs from each content
    buf.random_(0, 256)
    for name, fn in ops.items():
        out[name] = n * MiB / GiB / timed(fn, runs)
    return out


def cfg(path, size, seed=SEED, report=False):
    return WorkerConfig(paths=[path], block_size=MiB, file_size=size, num_threads=16,
                        integrity_check_salt=seed, integrity_check_kind=kernels.VERIFY_RANDOM,
                        block_variance_percent=100, verify_report=report)


def read(path, size, seed=SEED, report=False):
    with WorkerManager(cfg(path, size, seed, report)) as mgr:
        mgr.start_phase(BenchPhase.READFILES)
        t0 = time.perf_counter()
        try:
            mgr.wait_done(-1)
        except WorkerError:
            pass
        res = mgr.phase_results()
        t_report = time.perf_counter()
        num_extents = len(mgr.verify_report()) if report else 0
        report_sec = time.perf_counter() - t_report
        wall = t_report - t0
    rate = res["ops_total"]["bytes"] / GiB / (res["last_finish_usec"] / 1e6)
    return {"gib_per_s": round(rate, 3), "phase_wall_s": round(wall, 3),
            "report_merge_s": round(report_sec, 3), "extents": num_extents,
            "mismatch_bytes": res["verify_mismatch_bytes"], "bytes": res["ops_total"]["bytes"]}


def main():
    parser = argparse.ArgumentParser()
    parser.add_argument("--size-gib", type=int, default=16)
    parser.add_argument("--runs", type=int, default=3)
    parser.add_argument("--dir", default="/dev/shm")
    args = parser.parse_args()
    torch.cuda.set_device(0)
    info = gpu_info()

    for name, rate in kernel_rates(max(args.runs, 5)).items():
        print(json.dumps({"gpu": info, "kernel": name, "window_gib": 1, "gib_per_s": round(rate, 1)}),
              flush=True)

    size = args.size_gib * GiB
    workdir = tempfile.mkdtemp(prefix="elb_bench_report_", dir=args.dir)
    path = os.path.join(workdir, "f")
    try:
        with WorkerManager(cfg(path, size)) as mgr:
            mgr.run_phase(BenchPhase.CREATEFILES)
        for run in range(args.runs):
            for report in (False, True):
                print(json.dumps({"gpu": info, "read": "clean", "report": report, "run": run,
                                  **read(path, size, report=report)}), flush=True)
        # 1 % of the blocks damaged: one 4 KiB run in every 100th block
        fd = os.open(path, os.O_RDWR)
        try:
            for off in range(0, size, 100 * MiB):
                os.pwrite(fd, bytes(4096), off + 12345)
        finally:
            os.close(fd)
        for run in range(args.runs):
            print(json.dumps({"gpu": info, "read": "1pct_blocks_damaged", "report": True,
                              "run": run, **read(path, size, report=True)}), flush=True)
        # every block damaged: the bytes of another seed's content
        for run in range(args.runs):
            print(json.dumps({"gpu": info, "read": "all_blocks_damaged", "report": True,
                              "run": run, **read(path, size, seed=SEED + 1, report=True)}),
                  flush=True)
    finally:
        shutil.rmtree(workdir, ignore_errors=True)


if __name__ == "__main__":
    main()
