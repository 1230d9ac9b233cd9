"""--compressstats on the GPU: the LZ4 kernel's rate and the end-to-end cost of the option on
sequential reads.

Kernel: elb_lz4_chunks (the size-only path the worker runs) over a resident window of 4 GiB of
1 MiB blocks at K = 4 KiB, 64 KiB and 1 MiB, on random data (the fill of --verifyrand),
--blockvarpct 50 data and zeros (CUDA events, median of 5), next to the pinned host-to-device
copy rate of the same job.
Per batch: one launch over one 1 MiB block, as the worker makes it, 1024 batches captured in one
CUDA graph, at K = 4 KiB and 64 KiB, so that the per-launch cost that a window-sized launch hides
is measured.
End to end: a 16 GiB file in /dev/shm read sequentially with 1 MiB blocks and 16 threads, three
alternating runs without and with --compressstats 64K. Prints one JSON line per measurement and
the card's name, power limit and SM clock."""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from elbencho_b200 import BenchPhase, WorkerConfig, WorkerManager, kernels  # noqa: E402

KiB, MiB, GiB = 1 << 10, 1 << 20, 1 << 30


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def timed(fn, reps=5):
    times = []
    for _ in range(reps):
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        fn()
        stop.record()
        stop.synchronize()
        times.append(start.elapsed_time(stop) / 1e3)
    return statistics.median(times)


def copy_rate(window):
    host = torch.empty(window, dtype=torch.uint8).pin_memory()
    dev = torch.empty(window, dtype=torch.uint8, device="cuda")
    dev.copy_(host, non_blocking=True)
    return window / timed(lambda: dev.copy_(host, non_blocking=True)) / GiB


def fill(buf, kind, block):
    stream = torch.cuda.current_stream().cuda_stream
    if kind == "zero":
        buf.zero_()
        return
    pct = 100 if kind == "random" else 50
    for i in range(buf.numel() // block):
        kernels.fill_random(buf.data_ptr() + i * block, block, pct, 12345, i, stream)


def kernel_rates(window, block=MiB):
    buf = torch.empty(window, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    num_blocks = window // block
    raw = kernels.pack_block_descs([(buf.data_ptr() + i * block, block, i * block, 0)
                                    for i in range(num_blocks)])
    descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).pin_memory()
    counters = torch.zeros(4, dtype=torch.int64, device="cuda")
    rows = []
    for kind in ("random", "blockvar50", "zero"):
        fill(buf, kind, block)
        for k in (4 * KiB, 64 * KiB, MiB):
            shift, slots = k.bit_length() - 1, block // k

            def run():
                kernels.lz4_chunks(descs.data_ptr(), num_blocks, shift, slots,
                                   counters.data_ptr(), 0, 0, stream)

            run()
            counters.zero_()
            run()
            n, b, s, u = counters.cpu().tolist()
            t = timed(run)
            rows.append(dict(data=kind, chunk=k, lz4_gib_s=round(window / t / GiB, 1),
                             chunks=n, ratio=round(b / s, 2), incompressible=u))
    return rows


def batch_rates(num_batches=1024, batch=MiB):
    """per-batch cost: num_batches launches of one block each, replayed from a graph"""
    buf = torch.empty(num_batches * batch, dtype=torch.uint8, device="cuda")
    fill(buf, "random", batch)
    raw = kernels.pack_block_descs([(buf.data_ptr() + i * batch, batch, i * batch, 0)
                                    for i in range(num_batches)])
    descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).pin_memory()
    counters = torch.zeros(4, dtype=torch.int64, device="cuda")
    rows = []
    for k in (4 * KiB, 64 * KiB):
        shift, slots = k.bit_length() - 1, batch // k
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            stream = torch.cuda.current_stream().cuda_stream
            for b in range(num_batches):
                kernels.lz4_chunks(descs.data_ptr() + b * kernels.BLOCK_DESC_BYTES, 1, shift,
                                   slots, counters.data_ptr(), 0, 0, stream)
        g.replay()
        times = []
        for _ in range(5):
            start = torch.cuda.Event(enable_timing=True)
            stop = torch.cuda.Event(enable_timing=True)
            start.record()
            g.replay()
            stop.record()
            stop.synchronize()
            times.append(start.elapsed_time(stop) * 1e3 / num_batches)
        usec = statistics.median(times)
        rows.append(dict(per_batch=batch, chunk=k, lz4_usec=round(usec, 2),
                         batch_gib_s=round(batch / (usec / 1e6) / GiB, 1)))
    return rows


def end_to_end(size, threads, runs):
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    workdir = tempfile.mkdtemp(prefix="elb_compress_bench_", dir=base)
    path = os.path.join(workdir, "f")
    args = dict(paths=[path], file_size=size, block_size=MiB, num_threads=threads,
                block_variance_percent=50)
    try:
        with WorkerManager(WorkerConfig(**args)) as mgr:
            mgr.run_phase(BenchPhase.CREATEFILES)
        rates = {"off": [], "on": []}
        for _ in range(runs):
            for name, extra in (("off", {}), ("on", dict(compress_chunk=64 * KiB))):
                with WorkerManager(WorkerConfig(**args, **extra)) as mgr:
                    t = time.perf_counter()
                    res = mgr.run_phase(BenchPhase.READFILES)
                    rates[name].append(round(res["ops_total"]["bytes"] /
                                             (time.perf_counter() - t) / GiB, 2))
        return rates
    finally:
        shutil.rmtree(workdir, ignore_errors=True)


def main():
    parser = argparse.ArgumentParser()
    parser.add_argument("--window", type=int, default=4 * GiB)
    parser.add_argument("--size", type=int, default=16 * GiB)
    parser.add_argument("--threads", type=int, default=16)
    parser.add_argument("--runs", type=int, default=3)
    parser.add_argument("--skip-e2e", action="store_true")
    args = parser.parse_args()
    print(json.dumps(dict(card=card())), flush=True)
    print(json.dumps(dict(pinned_h2d_gib_s=round(copy_rate(min(args.window, GiB)), 1))),
          flush=True)
    for row in kernel_rates(args.window):
        print(json.dumps(row), flush=True)
    for row in batch_rates():
        print(json.dumps(row), flush=True)
    if not args.skip_e2e:
        print(json.dumps(dict(e2e_read_gib_s=end_to_end(args.size, args.threads, args.runs))),
              flush=True)
    print(json.dumps(dict(card_after=card())), flush=True)


if __name__ == "__main__":
    main()
