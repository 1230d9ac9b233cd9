"""--reducestats on the GPU: the rate of its launches and the end-to-end cost of the option on
sequential reads.

Kernels: the BLAKE3 chunk launch, elb_reduce_insert and elb_reduce_lz4 (the three launches of a
batch) over a resident window of 4 GiB of 1 MiB blocks at K = 64 KiB, on --dedupepct 0, 50 and
100 data with a 64 KiB grain and --blockvarpct 50 (the fill of the worker), the table cleared
before each run (CUDA events, median of 5), next to the pinned host-to-device copy rate of the
same job. The LZ4 launch is also timed alone.
Per batch: the three launches over one 1 MiB block, as the worker makes them, 1024 batches
captured in one CUDA graph, at K = 4 KiB and 64 KiB on --dedupepct 0 data.
End to end: a 16 GiB file in /dev/shm written with --dedupepct 0 and 90 (64 KiB grains,
--blockvarpct 50), read sequentially with 1 MiB blocks and 16 threads, three alternating runs
without and with --reducestats 64K. Prints one JSON line per measurement and the card's name,
power limit and SM clock."""
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
GRAIN_SHIFT = 16


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


def fill(buf, dedupe_pct, block):
    stream = torch.cuda.current_stream().cuda_stream
    for i in range(buf.numel() // block):
        kernels.fill_dedupe_grain(buf.data_ptr() + i * block, block, i * block, GRAIN_SHIFT, 50,
                                  dedupe_pct, 12345, 1, stream)


class Reduce:
    """a reduce table and the buffers of the three launches over num_descs descriptors"""

    def __init__(self, descs, num_descs, shift, slots, num_chunks):
        entries = 1024
        while entries < 2 * num_chunks:
            entries *= 2
        self.descs, self.num_descs, self.shift, self.slots = descs, num_descs, shift, slots
        self.entries = entries
        self.table = torch.zeros(entries * (16 + kernels.REDUCE_PAYLOAD_BYTES), dtype=torch.uint8,
                                 device="cuda")
        self.counters = torch.zeros(kernels.REDUCE_COUNTERS_BYTES, dtype=torch.uint8,
                                    device="cuda")
        self.digests = torch.empty(num_descs * slots * 32, dtype=torch.uint8, device="cuda")
        self.marks = torch.empty(num_descs * slots, dtype=torch.int64, device="cuda")

    def clear(self):
        self.table.zero_()
        self.counters.zero_()

    def launch(self, desc_ptr, num_descs, stream, lz4=True, hash_insert=True):
        keys, payloads = self.table.data_ptr(), self.table.data_ptr() + 16 * self.entries
        if hash_insert:
            kernels.blake3_chunks(desc_ptr, 0, num_descs, self.shift, self.slots,
                                  self.digests.data_ptr(), stream=stream)
            kernels.reduce_insert(desc_ptr, num_descs, self.shift, self.slots,
                                  self.digests.data_ptr(), keys, self.entries,
                                  self.counters.data_ptr(), self.marks.data_ptr(), stream)
        if lz4:
            kernels.reduce_lz4(desc_ptr, num_descs, self.shift, self.slots, self.marks.data_ptr(),
                               payloads, stream)

    def counts(self):
        kernels.reduce_sum(self.table.data_ptr(), self.table.data_ptr() + 16 * self.entries,
                           self.entries, self.counters.data_ptr(),
                           torch.cuda.current_stream().cuda_stream)
        return kernels.reduce_counters(self.counters.cpu().numpy().tobytes())


def kernel_rates(window, block=MiB, k=64 * KiB):
    buf = torch.empty(window, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    num_blocks = window // block
    raw = kernels.pack_block_descs([(buf.data_ptr() + i * block, block, i * block, 0)
                                    for i in range(num_blocks)])
    descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).pin_memory()
    shift, slots = k.bit_length() - 1, block // k
    red = Reduce(descs, num_blocks, shift, slots, window // k)
    rows = []
    for dedupe_pct in (0, 50, 100):
        fill(buf, dedupe_pct, block)

        def run():
            red.clear()
            red.launch(descs.data_ptr(), num_blocks, stream)

        run()
        n, b, d, u, s, _ = red.counts()
        t_all = timed(run)

        def run_lz4():  # (the marks of the last insert)
            red.launch(descs.data_ptr(), num_blocks, stream, hash_insert=False)

        t_lz4 = timed(run_lz4)
        rows.append(dict(dedupepct=dedupe_pct, chunk=k, chunks=n, distinct=d,
                         dedupe=round(b / u, 2), compress=round(u / s, 2),
                         launches_gib_s=round(window / t_all / GiB, 1),
                         lz4_ms=round(t_lz4 * 1e3, 2), all_ms=round(t_all * 1e3, 2)))
    return rows


def batch_rates(num_batches=1024, batch=MiB):
    """per-batch cost: the three launches of one block per batch, replayed from a graph"""
    buf = torch.empty(num_batches * batch, dtype=torch.uint8, device="cuda")
    fill(buf, 0, batch)
    raw = kernels.pack_block_descs([(buf.data_ptr() + i * batch, batch, i * batch, 0)
                                    for i in range(num_batches)])
    descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).pin_memory()
    rows = []
    for k in (4 * KiB, 64 * KiB):
        shift, slots = k.bit_length() - 1, batch // k
        red = Reduce(descs, 1, shift, slots, num_batches * slots)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            stream = torch.cuda.current_stream().cuda_stream
            for b in range(num_batches):
                red.launch(descs.data_ptr() + b * kernels.BLOCK_DESC_BYTES, 1, stream)
        times = []
        for _ in range(6):
            red.clear()
            torch.cuda.synchronize()
            start = torch.cuda.Event(enable_timing=True)
            stop = torch.cuda.Event(enable_timing=True)
            start.record()
            g.replay()
            stop.record()
            stop.synchronize()
            times.append(start.elapsed_time(stop) * 1e3 / num_batches)
        usec = statistics.median(times[1:])
        rows.append(dict(per_batch=batch, chunk=k, reduce_usec=round(usec, 2),
                         batch_gib_s=round(batch / (usec / 1e6) / GiB, 1)))
    return rows


def end_to_end(size, threads, runs, dedupe_pct):
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    workdir = tempfile.mkdtemp(prefix="elb_reduce_bench_", dir=base)
    path = os.path.join(workdir, "f")
    args = dict(paths=[path], file_size=size, block_size=MiB, num_threads=threads)
    try:
        with WorkerManager(WorkerConfig(**args, integrity_check_salt=7,
                                        integrity_check_kind=kernels.VERIFY_RANDOM,
                                        verify_random_grain=1 << GRAIN_SHIFT,
                                        dedupe_percent=dedupe_pct,
                                        block_variance_percent=50)) as mgr:
            mgr.run_phase(BenchPhase.CREATEFILES)
        rates = {"off": [], "on": []}
        line = None
        for _ in range(runs):
            for name, extra in (("off", {}), ("on", dict(reduce_chunk=64 * KiB))):
                with WorkerManager(WorkerConfig(**args, **extra)) as mgr:
                    t = time.perf_counter()
                    res = mgr.run_phase(BenchPhase.READFILES)
                    rates[name].append(round(res["ops_total"]["bytes"] /
                                             (time.perf_counter() - t) / GiB, 2))
                    if extra:
                        line = kernels.reduce_line(64 * KiB, *mgr.reduce_stats())
        return dict(dedupepct=dedupe_pct, e2e_read_gib_s=rates, line=line)
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
        for dedupe_pct in (0, 90):
            print(json.dumps(end_to_end(args.size, args.threads, args.runs, dedupe_pct)),
                  flush=True)
    print(json.dumps(dict(card_after=card())), flush=True)


if __name__ == "__main__":
    main()
