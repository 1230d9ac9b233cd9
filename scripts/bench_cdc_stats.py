"""--cdcstats on the GPU: the rate of its launches and the end-to-end cost of the option on
sequential reads.

Kernels: elb_cdc_cut alone, and elb_cdc_cut plus elb_cdc_hash_insert (the two launches of a batch),
over a resident window of 4 GiB of 1 MiB blocks at AVG 4K, 16K and 64K, on random data,
--blockvarpct 50 data (the fill of the worker) and zero data, the table cleared before each run
(CUDA events, median of 5), next to the pinned host-to-device copy rate of the same job.
Per batch: the two launches over one 1 MiB block, as the worker makes them, 1024 batches captured
in one CUDA graph, at AVG 16K on random data.
End to end: a 16 GiB file in /dev/shm written with --blockvarpct 100, read sequentially with 1 MiB
blocks and 16 threads, three alternating runs without and with --cdcstats 16K. Prints one JSON
line per measurement and the card's name, power limit and SM clock."""
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
    """random (--blockvarpct 100), blockvar50 (--blockvarpct 50) or zero blocks"""
    if kind == "zero":
        buf.zero_()
        return
    stream = torch.cuda.current_stream().cuda_stream
    pct = 100 if kind == "random" else 50
    for i in range(buf.numel() // block):
        kernels.fill_dedupe_grain(buf.data_ptr() + i * block, block, i * block, 16, pct, 0,
                                  12345, 1, stream)


class Cdc:
    """a CDC table and the buffers of the two launches over num_descs descriptors"""

    def __init__(self, num_descs, avg, slots, num_chunks):
        entries = 1024
        while entries < 2 * num_chunks:
            entries *= 2
        self.shift, self.slots, self.entries = avg.bit_length() - 1, slots, entries
        self.table = torch.zeros(entries * (16 + kernels.REDUCE_PAYLOAD_BYTES), dtype=torch.uint8,
                                 device="cuda")
        self.counters = torch.zeros(kernels.REDUCE_COUNTERS_BYTES, dtype=torch.uint8,
                                    device="cuda")
        self.counts = torch.empty(num_descs, dtype=torch.int32, device="cuda")
        self.ends = torch.empty(num_descs * slots, dtype=torch.int64, device="cuda")

    def clear(self):
        self.table.zero_()
        self.counters.zero_()

    def launch(self, desc_ptr, num_descs, stream, hash_insert=True, offset=0):
        kernels.cdc_cut(desc_ptr, num_descs, self.shift, self.slots,
                        self.counts.data_ptr() + 4 * offset,
                        self.ends.data_ptr() + 8 * offset * self.slots, stream)
        if hash_insert:
            kernels.cdc_hash_insert(desc_ptr, num_descs, self.shift, self.slots,
                                    self.counts.data_ptr() + 4 * offset,
                                    self.ends.data_ptr() + 8 * offset * self.slots, 0,
                                    self.table.data_ptr(),
                                    self.table.data_ptr() + 16 * self.entries, self.entries,
                                    self.counters.data_ptr(), stream)

    def stats(self):
        kernels.reduce_sum(self.table.data_ptr(), self.table.data_ptr() + 16 * self.entries,
                           self.entries, self.counters.data_ptr(),
                           torch.cuda.current_stream().cuda_stream)
        return kernels.reduce_counters(self.counters.cpu().numpy().tobytes())


def pinned_descs(buf, num_blocks, block):
    raw = kernels.pack_block_descs([(buf.data_ptr() + i * block, block, i * block, 0)
                                    for i in range(num_blocks)])
    return torch.frombuffer(bytearray(raw), dtype=torch.uint8).pin_memory()


def kernel_rates(window, block=MiB):
    buf = torch.empty(window, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    num_blocks = window // block
    descs = pinned_descs(buf, num_blocks, block)
    rows = []
    for kind in ("random", "blockvar50", "zero"):
        fill(buf, kind, block)
        for avg in (4 * KiB, 16 * KiB, 64 * KiB):
            slots = block // (avg // 4)
            cdc = Cdc(num_blocks, avg, slots, window // (avg // 4))

            def run(hash_insert=True):
                cdc.clear()
                cdc.launch(descs.data_ptr(), num_blocks, stream, hash_insert)

            run()
            n, b, d, u, _, overflow = cdc.stats()
            t_cut = timed(lambda: run(False))
            t_all = timed(run)
            rows.append(dict(data=kind, avg=avg, chunks=n, distinct=d, mean=b // max(n, 1),
                             dedupe=round(b / u, 2), overflow=overflow,
                             cut_gib_s=round(window / t_cut / GiB, 1),
                             cut_ms=round(t_cut * 1e3, 2),
                             both_gib_s=round(window / t_all / GiB, 1),
                             both_ms=round(t_all * 1e3, 2)))
            del cdc
    return rows


def batch_rates(num_batches=1024, batch=MiB, avg=16 * KiB):
    """per-batch cost: the two launches of one block per batch, replayed from a graph"""
    buf = torch.empty(num_batches * batch, dtype=torch.uint8, device="cuda")
    fill(buf, "random", batch)
    descs = pinned_descs(buf, num_batches, batch)
    cdc = Cdc(num_batches, avg, batch // (avg // 4), num_batches * batch // (avg // 4))
    rows = []
    for hash_insert in (False, True):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            stream = torch.cuda.current_stream().cuda_stream
            for b in range(num_batches):
                cdc.launch(descs.data_ptr() + b * kernels.BLOCK_DESC_BYTES, 1, stream,
                           hash_insert, offset=b)
        times = []
        for _ in range(6):
            cdc.clear()
            torch.cuda.synchronize()
            start = torch.cuda.Event(enable_timing=True)
            stop = torch.cuda.Event(enable_timing=True)
            start.record()
            g.replay()
            stop.record()
            stop.synchronize()
            times.append(start.elapsed_time(stop) * 1e3 / num_batches)
        usec = statistics.median(times[1:])
        rows.append(dict(per_batch=batch, avg=avg, launches="cut+hash_insert" if hash_insert
                         else "cut", usec=round(usec, 2),
                         batch_gib_s=round(batch / (usec / 1e6) / GiB, 2)))
    return rows


def end_to_end(size, threads, runs):
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    workdir = tempfile.mkdtemp(prefix="elb_cdc_bench_", dir=base)
    path = os.path.join(workdir, "f")
    args = dict(paths=[path], file_size=size, block_size=MiB, num_threads=threads)
    try:
        with WorkerManager(WorkerConfig(**args, block_variance_percent=100)) as mgr:
            mgr.run_phase(BenchPhase.CREATEFILES)
        rates = {"off": [], "on": []}
        line = None
        for _ in range(runs):
            for name, extra in (("off", {}), ("on", dict(cdc_avg=16 * KiB))):
                with WorkerManager(WorkerConfig(**args, **extra)) as mgr:
                    t = time.perf_counter()
                    res = mgr.run_phase(BenchPhase.READFILES)
                    rates[name].append(round(res["ops_total"]["bytes"] /
                                             (time.perf_counter() - t) / GiB, 2))
                    if extra:
                        line = kernels.cdc_line(16 * KiB, *mgr.cdc_stats())
        return dict(e2e_read_gib_s=rates, line=line)
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
        print(json.dumps(end_to_end(args.size, args.threads, args.runs)), flush=True)
    print(json.dumps(dict(card_after=card())), flush=True)


if __name__ == "__main__":
    main()
