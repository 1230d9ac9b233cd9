"""Rates of --verifyrandgrain on one GPU: K5 fill_random_grain against K3 fill_random and K6
verify_random_grain against K4 verify_random on a resident window for each launch shape, grain
size and pct; K6 against K4 in their stage-in + verify forms over PCIe; and one file written with
1 MiB blocks, read back sequentially and with 4 KiB random reads at iodepth 64 (BASELINE config 2's
shape), under --verifyrandgrain and under --verify. Old and new alternate within one process; the
card's name, power limit and max SM clock are read in the same run.

    python scripts/bench_verify_random_grain.py [--window-gib 4] [--file-gib 16] [--threads 16]
                                                [--dir /dev/shm] [--reps 3] [--out result.json]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

from elbencho_b200 import BenchPhase, WorkerConfig, WorkerManager, kernels  # noqa: E402
from scripts.bench_verify_random import card_info, time_launches  # noqa: E402

GiB, MiB, KiB = 1 << 30, 1 << 20, 1 << 10
SEED, FILE_KEY = 0xC0FFEE, 3
SHAPES = {"tiled_1MiB": (MiB, "hinted"), "warp_4KiB": (4 * KiB, "hinted"),
          "persistent_1MiB_unhinted": (MiB, "none")}
GRAIN_SHIFTS = {"4KiB": 12, "64KiB": 16, "1MiB": 20}


def descs_for(buf, window, block, grain_mode, device):
    """grain mode: fileKey in the counter field, file position = window offset"""
    raw = kernels.pack_block_descs(
        (buf.data_ptr() + off, block, off, FILE_KEY if grain_mode else off // block)
        for off in range(0, window, block))
    t = torch.frombuffer(bytearray(raw), dtype=torch.uint8)
    return t.to(device) if device is not None else t.pin_memory()


def gbps(window, vals):
    return [round(window / v / 1e6, 1) for v in vals]


def resident(window, reps, pct):
    s = torch.cuda.current_stream().cuda_stream
    buf = torch.empty(window, dtype=torch.uint8, device="cuda")
    counters = torch.zeros(kernels.DEVCTR_NUM, dtype=torch.int64, device="cuda")
    out = {}
    for name, (block, hinting) in SHAPES.items():
        n = window // block
        hints = dict(total_bytes=window, max_block_len=block) if hinting == "hinted" else {}
        per_block = descs_for(buf, window, block, False, "cuda")
        grain = descs_for(buf, window, block, True, "cuda")
        res = torch.empty(2 * n, dtype=torch.int64, device="cuda")
        init_ms = time_launches(lambda: kernels.verify_results_init(res.data_ptr(), n, s), 20)
        runs = {"K3": [], "K4": []}
        runs.update({"K5_" + g: [] for g in GRAIN_SHIFTS})
        runs.update({"K6_" + g: [] for g in GRAIN_SHIFTS})
        for _ in range(reps):
            runs["K3"].append(time_launches(lambda: kernels.fill_random_batch(
                per_block.data_ptr(), n, pct, SEED, 0, s, **hints), 20))
            runs["K4"].append(time_launches(lambda: kernels.verify_random_batch(
                per_block.data_ptr(), n, pct, SEED, res.data_ptr(), counters.data_ptr(), s,
                **hints), 20) - init_ms)
            assert int(counters[kernels.DEVCTR_VERIFY_MISMATCH_BYTES]) == 0
            for g, shift in GRAIN_SHIFTS.items():
                runs["K5_" + g].append(time_launches(lambda: kernels.fill_random_grain_batch(
                    grain.data_ptr(), n, shift, pct, SEED, 0, s, **hints), 20))
                runs["K6_" + g].append(time_launches(lambda: kernels.verify_random_grain_batch(
                    grain.data_ptr(), n, shift, pct, SEED, res.data_ptr(), counters.data_ptr(), s,
                    **hints), 20) - init_ms)
                assert int(counters[kernels.DEVCTR_VERIFY_MISMATCH_BYTES]) == 0
            # (each K4 / K6 run above verified the content of the fill just before it)
            kernels.fill_random_batch(per_block.data_ptr(), n, pct, SEED, 0, s, **hints)
        cell = {k: dict(ms=[round(v, 4) for v in vals], gbps=gbps(window, vals))
                for k, vals in runs.items()}
        for g in GRAIN_SHIFTS:
            cell["K5_%s_over_K3" % g] = round(min(runs["K3"]) / min(runs["K5_" + g]), 3)
            cell["K6_%s_over_K4" % g] = round(min(runs["K4"]) / min(runs["K6_" + g]), 3)
        out[name] = cell
    del buf
    torch.cuda.empty_cache()
    return out


def staged(window, reps):
    """stage-in + verify over PCIe from pinned host memory, 1 MiB blocks, tiled shape"""
    s = torch.cuda.current_stream().cuda_stream
    dev = torch.empty(window, dtype=torch.uint8, device="cuda")
    host = torch.empty(window, dtype=torch.uint8).pin_memory()
    delta = host.data_ptr() - dev.data_ptr()
    n = window // MiB
    hints = dict(total_bytes=window, max_block_len=MiB)
    per_block = descs_for(dev, window, MiB, False, None)
    grain = descs_for(dev, window, MiB, True, None)
    dev_res = torch.empty(2 * n, dtype=torch.int64, device="cuda")
    host_res = torch.empty(2 * n, dtype=torch.int64).pin_memory()
    ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
    kernels.verify_results_init(dev_res.data_ptr(), n, s)
    runs = {"K4": [], "K6_64KiB": []}
    for _ in range(reps):
        kernels.fill_random_staged(per_block.data_ptr(), n, 100, SEED, delta, 0, s, **hints)
        runs["K4"].append(time_launches(lambda: kernels.verify_random_staged(
            per_block.data_ptr(), n, 100, SEED, delta, dev_res.data_ptr(), host_res.data_ptr(),
            ticket.data_ptr(), 0, s, **hints), 5))
        assert all(v == 0 for v in host_res.tolist()[0::2])
        kernels.fill_random_grain_staged(grain.data_ptr(), n, 16, 100, SEED, delta, 0, s, **hints)
        runs["K6_64KiB"].append(time_launches(lambda: kernels.verify_random_grain_staged(
            grain.data_ptr(), n, 16, 100, SEED, delta, dev_res.data_ptr(), host_res.data_ptr(),
            ticket.data_ptr(), 0, s, **hints), 5))
        assert all(v == 0 for v in host_res.tolist()[0::2])
    return {k: dict(gib_per_s=[round(window / GiB / (v / 1e3), 2) for v in vals])
            for k, vals in runs.items()}


def end_to_end(file_bytes, threads, directory, reps, rand_bytes):
    """one file written with 1 MiB blocks, then read sequentially with 1 MiB blocks and with 4 KiB
    random reads at iodepth 64: --verifyrandgrain 64K against --verify, GiB/s of each phase"""
    out = {"verify": [], "verifyrandgrain_64K": []}
    workdir = tempfile.mkdtemp(prefix="elb_vrg_bench_", dir=directory)
    try:
        path = os.path.join(workdir, "f")
        for _ in range(reps):
            for name, kind, grain in (("verify", kernels.VERIFY_PATTERN, 0),
                                      ("verifyrandgrain_64K", kernels.VERIFY_RANDOM, 64 * KiB)):
                common = dict(paths=[path], num_threads=threads, file_size=file_bytes,
                              integrity_check_salt=SEED, integrity_check_kind=kind,
                              block_variance_percent=100 if grain else 0,
                              verify_random_grain=grain)
                rates = {}
                for label, phase, extra in (
                        ("write_1M", BenchPhase.CREATEFILES, dict(block_size=MiB)),
                        ("read_seq_1M", BenchPhase.READFILES, dict(block_size=MiB)),
                        ("read_rand_4K_qd64", BenchPhase.READFILES,
                         dict(block_size=4 * KiB, use_random_offsets=True, rand_offset_seed=7,
                              io_depth=64, random_amount=rand_bytes))):
                    with WorkerManager(WorkerConfig(**common, **extra)) as mgr:
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
    p.add_argument("--rand-gib", type=float, default=2.0,
                   help="bytes of the 4 KiB random read phase (--randamount)")
    p.add_argument("--threads", type=int, default=16)
    p.add_argument("--dir", default="/dev/shm")
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--skip-e2e", action="store_true")
    p.add_argument("--out", default=None)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_verify_random_grain.py needs a CUDA device")
    file_bytes = int(args.file_gib * GiB) // MiB * MiB
    if not args.skip_e2e and file_bytes > shutil.disk_usage(args.dir).free - GiB:
        raise SystemExit("%s has too little free space for a %.1f GiB file" % (
            args.dir, file_bytes / GiB))
    t0 = time.time()
    window = int(args.window_gib * GiB)
    result = dict(card=card_info(), window_gib=args.window_gib,
                  resident_pct100=resident(window, args.reps, 100),
                  resident_pct50=resident(window, args.reps, 50),
                  staged_tiled_1MiB=staged(int(args.staged_gib * GiB), args.reps))
    if not args.skip_e2e:
        result["end_to_end"] = dict(file_gib=file_bytes / GiB, threads=args.threads,
                                    rand_gib=args.rand_gib,
                                    runs=end_to_end(file_bytes, args.threads, args.dir, args.reps,
                                                    int(args.rand_gib * GiB)))
    result["seconds"] = round(time.time() - t0, 1)
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
