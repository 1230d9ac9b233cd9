"""--cdcreducestats on the GPU: the rate of its launches and the end-to-end cost of the option on
sequential reads.

Kernels: elb_cdc_cut plus elb_cdc_hash_insert_marks (what --cdcstats launches, with marks), and
those plus elb_cdc_lz4 (the three launches of a batch), over a resident window of 4 GiB of 1 MiB
blocks at AVG 4K, 16K and 64K, on random data, --blockvarpct 50 data (the fill of the worker) and
zero data, the table cleared before each run (CUDA events, median of 5), next to the pinned
host-to-device copy rate of the same job.
Per batch: the three launches over one 1 MiB block, as the worker makes them, 1024 batches
captured in one CUDA graph, at AVG 16K and 256K on random data.
End to end: a 16 GiB file in /dev/shm written with --blockvarpct 100, read sequentially with 1 MiB
blocks and 16 threads, three alternating runs each without an option, with --cdcstats 16K and with
--cdcreducestats 16K. Prints one JSON line per measurement and the card's name, power limit and SM
clock."""
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


class CdcReduce:
    """a CDC reduce table and the buffers of the three launches over num_descs descriptors"""

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
        self.marks = torch.empty(num_descs * slots, dtype=torch.int64, device="cuda")

    def clear(self):
        self.table.zero_()
        self.counters.zero_()

    def launch(self, desc_ptr, num_descs, stream, lz4=True, offset=0):
        counts = self.counts.data_ptr() + 4 * offset
        ends = self.ends.data_ptr() + 8 * offset * self.slots
        marks = self.marks.data_ptr() + 8 * offset * self.slots
        payloads = self.table.data_ptr() + 16 * self.entries
        kernels.cdc_cut(desc_ptr, num_descs, self.shift, self.slots, counts, ends, stream)
        kernels.cdc_hash_insert_marks(desc_ptr, num_descs, self.shift, self.slots, counts, ends, 0,
                                      self.table.data_ptr(), payloads, self.entries,
                                      self.counters.data_ptr(), marks, stream)
        if lz4:
            kernels.cdc_lz4(desc_ptr, num_descs, self.shift, self.slots, counts, ends, marks,
                            payloads, stream)

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
            cdc = CdcReduce(num_blocks, avg, slots, window // (avg // 4))

            def run(lz4=True):
                cdc.clear()
                cdc.launch(descs.data_ptr(), num_blocks, stream, lz4)

            run()
            n, b, d, u, s, overflow = cdc.stats()
            t_insert = timed(lambda: run(False))
            t_all = timed(run)
            rows.append(dict(data=kind, avg=avg, chunks=n, distinct=d, mean=b // max(n, 1),
                             dedupe=round(b / u, 2), compress=round(u / s, 2),
                             overflow=overflow,
                             cut_insert_gib_s=round(window / t_insert / GiB, 1),
                             cut_insert_ms=round(t_insert * 1e3, 2),
                             all_gib_s=round(window / t_all / GiB, 1),
                             all_ms=round(t_all * 1e3, 2)))
            del cdc
    return rows


def batch_rates(num_batches=1024, batch=MiB):
    """per-batch cost: the three launches of one block per batch, replayed from a graph"""
    buf = torch.empty(num_batches * batch, dtype=torch.uint8, device="cuda")
    fill(buf, "random", batch)
    descs = pinned_descs(buf, num_batches, batch)
    rows = []
    for avg in (16 * KiB, 256 * KiB):
        cdc = CdcReduce(num_batches, avg, batch // (avg // 4), num_batches * batch // (avg // 4))
        for lz4 in (False, True):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                stream = torch.cuda.current_stream().cuda_stream
                for b in range(num_batches):
                    cdc.launch(descs.data_ptr() + b * kernels.BLOCK_DESC_BYTES, 1, stream, lz4,
                               offset=b)
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
            rows.append(dict(per_batch=batch, avg=avg, launches="cut+insert+lz4" if lz4
                             else "cut+insert", usec=round(usec, 2),
                             batch_gib_s=round(batch / (usec / 1e6) / GiB, 2)))
            del g
        del cdc
    return rows


def end_to_end(size, threads, runs):
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    workdir = tempfile.mkdtemp(prefix="elb_cdc_reduce_bench_", dir=base)
    path = os.path.join(workdir, "f")
    args = dict(paths=[path], file_size=size, block_size=MiB, num_threads=threads)
    try:
        with WorkerManager(WorkerConfig(**args, block_variance_percent=100)) as mgr:
            mgr.run_phase(BenchPhase.CREATEFILES)
        options = (("off", {}), ("cdcstats", dict(cdc_avg=16 * KiB)),
                   ("cdcreducestats", dict(cdc_reduce_avg=16 * KiB)))
        rates = {name: [] for name, _ in options}
        line = None
        for _ in range(runs):
            for name, extra in options:
                with WorkerManager(WorkerConfig(**args, **extra)) as mgr:
                    t = time.perf_counter()
                    res = mgr.run_phase(BenchPhase.READFILES)
                    rates[name].append(round(res["ops_total"]["bytes"] /
                                             (time.perf_counter() - t) / GiB, 2))
                    if name == "cdcreducestats":
                        line = kernels.cdc_reduce_line(16 * KiB, *mgr.cdc_reduce_stats())
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
