"""Rates of --verifyrand against --verify on one GPU: the K4 verify_random kernel against K2
verify_pattern on a resident window for each launch shape, their stage-in + verify forms over PCIe,
and a write + read of one file through the worker. Old and new alternate (K2, K4, K2, K4, ...)
within one process; the card's name, power limit and max SM clock are read in the same run.

    python scripts/bench_verify_random.py [--window-gib 4] [--file-gib 16] [--threads 16]
                                          [--dir /dev/shm] [--reps 3] [--out result.json]
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

from elbencho_b200 import BenchPhase, WorkerConfig, WorkerManager, kernels  # noqa: E402

GiB, MiB, KiB = 1 << 30, 1 << 20, 1 << 10
DATASHEET_BPS = 3.35e12  # H100 SXM HBM3
SALT, SEED = 1, 0xC0FFEE


def card_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout
    name, power, clock = [f.strip() for f in out.splitlines()[0].split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def descs_for(buf, window, block, device):
    raw = kernels.pack_block_descs((buf.data_ptr() + off, block, off, off // block)
                                   for off in range(0, window, block))
    t = torch.frombuffer(bytearray(raw), dtype=torch.uint8)
    return t.to(device) if device is not None else t.pin_memory()


def time_launches(launch, iters):
    """ms per launch from CUDA events around iters launches (after 3 warm-up launches)"""
    for _ in range(3):
        launch()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        launch()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def resident(window, reps, pct=100, shape_names=None):
    """K2 / K4 (K3 content of pct) over a resident window: GB/s and share of the data sheet, per
    shape"""
    s = torch.cuda.current_stream().cuda_stream
    buf = torch.empty(window, dtype=torch.uint8, device="cuda")
    counters = torch.zeros(kernels.DEVCTR_NUM, dtype=torch.int64, device="cuda")
    shapes = {"tiled_1MiB": (MiB, dict(total_bytes=window, max_block_len=MiB)),
              "warp_4KiB": (4 * KiB, dict(total_bytes=window, max_block_len=4 * KiB)),
              "persistent_1MiB_unhinted": (MiB, {})}
    out = {}
    for name, (block, hints) in shapes.items():
        if shape_names and name not in shape_names:
            continue
        n = window // block
        descs = descs_for(buf, window, block, "cuda")
        res = torch.empty(2 * n, dtype=torch.int64, device="cuda")
        init_ms = time_launches(lambda: kernels.verify_results_init(res.data_ptr(), n, s), 20)
        runs = {"verify_pattern": [], "verify_random": []}
        for _ in range(reps):
            kernels.fill_pattern_batch(descs.data_ptr(), n, SALT, 0, s, **hints)
            ms = time_launches(lambda: kernels.verify_pattern_batch(
                descs.data_ptr(), n, SALT, res.data_ptr(), counters.data_ptr(), s, **hints), 20)
            runs["verify_pattern"].append(ms - init_ms)
            assert int(counters[kernels.DEVCTR_VERIFY_MISMATCH_BYTES]) == 0
            kernels.fill_random_batch(descs.data_ptr(), n, pct, SEED, 0, s, **hints)
            ms = time_launches(lambda: kernels.verify_random_batch(
                descs.data_ptr(), n, pct, SEED, res.data_ptr(), counters.data_ptr(), s,
                **hints), 20)
            runs["verify_random"].append(ms - init_ms)
            assert int(counters[kernels.DEVCTR_VERIFY_MISMATCH_BYTES]) == 0
        out[name] = {k: dict(ms=[round(v, 4) for v in vals],
                             gbps=[round(window / v / 1e6, 1) for v in vals],
                             datasheet_fraction=[round(window / v / 1e-3 / DATASHEET_BPS, 3)
                                                 for v in vals])
                     for k, vals in runs.items()}
        out[name]["k4_over_k2"] = round(min(runs["verify_pattern"]) /
                                        min(runs["verify_random"]), 3)
    del buf
    torch.cuda.empty_cache()
    return out


def staged(window, reps, hinted):
    """stage-in + verify over PCIe from pinned host memory, 1 MiB blocks: tiled shape (hinted) or
    the persistent one (no size hints)"""
    s = torch.cuda.current_stream().cuda_stream
    dev = torch.empty(window, dtype=torch.uint8, device="cuda")
    host = torch.empty(window, dtype=torch.uint8).pin_memory()
    delta = host.data_ptr() - dev.data_ptr()
    n = window // MiB
    hints = dict(total_bytes=window, max_block_len=MiB) if hinted else {}
    descs = descs_for(dev, window, MiB, None)
    dev_res = torch.empty(2 * n, dtype=torch.int64, device="cuda")
    host_res = torch.empty(2 * n, dtype=torch.int64).pin_memory()
    ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
    kernels.verify_results_init(dev_res.data_ptr(), n, s)
    runs = {"verify_pattern": [], "verify_random": []}
    for _ in range(reps):
        kernels.fill_pattern_staged(descs.data_ptr(), n, SALT, delta, 0, s, **hints)
        runs["verify_pattern"].append(time_launches(lambda: kernels.verify_pattern_staged(
            descs.data_ptr(), n, SALT, delta, dev_res.data_ptr(), host_res.data_ptr(),
            ticket.data_ptr(), 0, s, **hints), 5))
        assert all(v == 0 for v in host_res.tolist()[0::2])
        kernels.fill_random_staged(descs.data_ptr(), n, 100, SEED, delta, 0, s, **hints)
        runs["verify_random"].append(time_launches(lambda: kernels.verify_random_staged(
            descs.data_ptr(), n, 100, SEED, delta, dev_res.data_ptr(), host_res.data_ptr(),
            ticket.data_ptr(), 0, s, **hints), 5))
        assert all(v == 0 for v in host_res.tolist()[0::2])
    return {k: dict(gib_per_s=[round(window / GiB / (v / 1e3), 2) for v in vals])
            for k, vals in runs.items()}


def end_to_end(file_bytes, threads, directory, reps):
    """write + read of one file, --verify against --verifyrand, GiB/s of each phase"""
    out = {"verify": [], "verifyrand": []}
    workdir = tempfile.mkdtemp(prefix="elb_vr_bench_", dir=directory)
    try:
        path = os.path.join(workdir, "f")
        for _ in range(reps):
            for name, kind in (("verify", kernels.VERIFY_PATTERN),
                               ("verifyrand", kernels.VERIFY_RANDOM)):
                cfg = WorkerConfig(paths=[path], num_threads=threads, block_size=MiB,
                                   file_size=file_bytes, integrity_check_salt=SEED,
                                   integrity_check_kind=kind, block_variance_percent=100)
                rates = {}
                with WorkerManager(cfg) as mgr:
                    for phase, label in ((BenchPhase.CREATEFILES, "write"),
                                         (BenchPhase.READFILES, "read")):
                        res = mgr.run_phase(phase)
                        assert res["verify_mismatch_bytes"] == 0
                        usec = res["last_finish_usec"]
                        rates[label] = round(res["ops_total"]["bytes"] / GiB / (usec / 1e6), 2)
                out[name].append(rates)
                os.unlink(path)
    finally:
        shutil.rmtree(workdir, ignore_errors=True)
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--window-gib", type=float, default=4.0)
    p.add_argument("--staged-gib", type=float, default=1.0)
    p.add_argument("--file-gib", type=float, default=16.0)
    p.add_argument("--threads", type=int, default=16)
    p.add_argument("--dir", default="/dev/shm")
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--out", default=None)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_verify_random.py needs a CUDA device")
    file_bytes = int(args.file_gib * GiB) // MiB * MiB
    free = shutil.disk_usage(args.dir).free
    if file_bytes > free - GiB:
        raise SystemExit("%s has %.1f GiB free, the file needs %.1f GiB" % (
            args.dir, free / GiB, file_bytes / GiB))
    t0 = time.time()
    result = dict(card=card_info(),
                  resident=resident(int(args.window_gib * GiB), args.reps),
                  # a block of 4 KiB is one warp span: at 0 < pct < 100 every span straddles the
                  # random part and the constant remainder
                  resident_pct50=resident(int(args.window_gib * GiB), args.reps, pct=50,
                                          shape_names=("tiled_1MiB", "warp_4KiB")),
                  staged_tiled=staged(int(args.staged_gib * GiB), args.reps, True),
                  staged_persistent_unhinted=staged(int(args.staged_gib * GiB), args.reps,
                                                    False),
                  end_to_end=dict(file_gib=file_bytes / GiB, threads=args.threads,
                                  runs=end_to_end(file_bytes, args.threads, args.dir,
                                                  args.reps)))
    result["seconds"] = round(time.time() - t0, 1)
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
