"""--dedupestats on the GPU: the insert kernel next to the BLAKE3 chunk launch it follows, and the
end-to-end cost of the option on sequential reads.

Kernel: elb_blake3_chunks alone and followed by elb_dedupe_insert over a resident window of 4 GiB
of 1 MiB and 4 KiB blocks, at K = 4 KiB and 64 KiB, with 0 %, 50 % and 100 % duplicate chunks
(CUDA events, median of 5), next to the pinned host-to-device copy rate of the same job. The
duplicates are copies of many distinct chunks: at P % the last P % of the chunks repeat the others
in turn, and at 100 % every chunk repeats one of a pool of 4096, as --dedupepct data does.
Per batch: the launches as the worker makes them, one BLAKE3 launch (and one insert) per 1 MiB
batch of one block, 1024 batches captured in one CUDA graph, so that the per-launch cost that a
window-sized launch hides is measured.
End to end: a 16 GiB file in /dev/shm read sequentially with 1 MiB blocks, three alternating runs
without and with --dedupestats 64K. Prints one JSON line per measurement and the card's name,
power limit and SM clock."""
import argparse
import json
import os
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


def kernel_rates(window):
    buf = torch.randint(0, 256, (window,), dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    rows = []
    for block in (MiB, 4 * KiB):
        num_blocks = window // block
        raw = kernels.pack_block_descs([(buf.data_ptr() + i * block, block, i * block, 0)
                                        for i in range(num_blocks)])
        descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).pin_memory()
        for k in (4 * KiB, 64 * KiB):
            if k > block:
                continue  # (a chunk must lie inside one block)
            shift, slots = k.bit_length() - 1, max(block // k, 1)
            digests = torch.empty(num_blocks * slots * 32, dtype=torch.uint8, device="cuda")
            entries = 1 << max(10, (2 * (window // k) - 1).bit_length())
            table = torch.zeros(entries * 16, dtype=torch.uint8, device="cuda")
            counters = torch.zeros(32, dtype=torch.uint8, device="cuda")
            zero = kernels.dedupe_zero_digest(shift)
            for dup in (0, 50, 100):
                chunks = buf.view(window // k, k)
                torch.manual_seed(dup)
                chunks.copy_(torch.randint(0, 256, chunks.shape, dtype=torch.uint8,
                                           device="cuda"))
                num_chunks = window // k
                first_dup = min(num_chunks * (100 - dup) // 100 or 4096, num_chunks)
                if first_dup < num_chunks:
                    chunks[first_dup:] = chunks[torch.arange(first_dup, num_chunks,
                                                             device="cuda") % first_dup]

                def blake3():
                    kernels.blake3_chunks(descs.data_ptr(), 0, num_blocks, shift, slots,
                                          digests.data_ptr(), 0, 0, stream)

                def both():
                    table.zero_()
                    counters.zero_()
                    blake3()
                    kernels.dedupe_insert(descs.data_ptr(), num_blocks, shift, slots,
                                          digests.data_ptr(), table.data_ptr(), entries,
                                          counters.data_ptr(), zero, stream)

                def clear_only():
                    table.zero_()
                    counters.zero_()

                blake3(), both()
                t_b3 = timed(blake3)
                t_both = timed(both) - timed(clear_only)
                both()
                n, d, z, overflow = kernels.dedupe_counters(counters.cpu().numpy().tobytes())
                rows.append(dict(block=block, chunk=k, dup_pct=dup,
                                 blake3_gib_s=round(window / t_b3 / GiB, 1),
                                 blake3_insert_gib_s=round(window / t_both / GiB, 1),
                                 insert_share_pct=round(100 * (t_both - t_b3) / t_b3, 1),
                                 chunks=n, distinct=d, overflow=overflow))
    return rows


def batch_rates(num_batches=1024, batch=MiB):
    """per-batch cost: num_batches launches (pairs) of one block each, replayed from a graph"""
    buf = torch.randint(0, 256, (num_batches * batch,), dtype=torch.uint8, device="cuda")
    raw = kernels.pack_block_descs([(buf.data_ptr() + i * batch, batch, i * batch, 0)
                                    for i in range(num_batches)])
    descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).pin_memory()
    rows = []
    for k in (4 * KiB, 64 * KiB):
        shift, slots = k.bit_length() - 1, batch // k
        digests = torch.empty(num_batches * slots * 32, dtype=torch.uint8, device="cuda")
        entries = 1 << max(10, (2 * num_batches * slots - 1).bit_length())
        table = torch.zeros(entries * 16, dtype=torch.uint8, device="cuda")
        counters = torch.zeros(32, dtype=torch.uint8, device="cuda")
        zero = kernels.dedupe_zero_digest(shift)
        graphs = {}
        for name in ("blake3", "blake3_insert"):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                stream = torch.cuda.current_stream().cuda_stream
                for b in range(num_batches):
                    d = descs.data_ptr() + b * kernels.BLOCK_DESC_BYTES
                    kernels.blake3_chunks(d, 0, 1, shift, slots,
                                          digests.data_ptr() + b * slots * 32, 0, 0, stream)
                    if name == "blake3_insert":
                        kernels.dedupe_insert(d, 1, shift, slots,
                                              digests.data_ptr() + b * slots * 32,
                                              table.data_ptr(), entries, counters.data_ptr(),
                                              zero, stream)
            graphs[name] = g
        usec = {}
        for name, g in graphs.items():
            times = []
            for _ in range(5):
                table.zero_()
                start = torch.cuda.Event(enable_timing=True)
                stop = torch.cuda.Event(enable_timing=True)
                start.record()
                g.replay()
                stop.record()
                stop.synchronize()
                times.append(start.elapsed_time(stop) * 1e3 / num_batches)
            usec[name] = statistics.median(times)
        rows.append(dict(per_batch=batch, chunk=k, blake3_usec=round(usec["blake3"], 2),
                         blake3_insert_usec=round(usec["blake3_insert"], 2),
                         insert_usec=round(usec["blake3_insert"] - usec["blake3"], 2)))
    return rows


def end_to_end(size, threads, runs):
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    workdir = tempfile.mkdtemp(prefix="elb_dedupe_bench_", dir=base)
    path = os.path.join(workdir, "f")
    args = dict(paths=[path], file_size=size, block_size=MiB, num_threads=threads,
                block_variance_percent=100)
    try:
        with WorkerManager(WorkerConfig(**args)) as mgr:
            mgr.run_phase(BenchPhase.CREATEFILES)
        rates = {"off": [], "on": []}
        for _ in range(runs):
            for name, extra in (("off", {}), ("on", dict(dedupe_chunk=64 * KiB))):
                with WorkerManager(WorkerConfig(**args, **extra)) as mgr:
                    t = time.perf_counter()
                    res = mgr.run_phase(BenchPhase.READFILES)
                    rates[name].append(round(res["ops_total"]["bytes"] /
                                             (time.perf_counter() - t) / GiB, 2))
        return rates
    finally:
        import shutil
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
