"""Rates of --dedupepct on one GPU: K7 fill_dedupe_grain against K5 fill_random_grain and K8
verify_dedupe_grain against K6 verify_random_grain on a resident window, for each launch shape,
grain size, dedupe percent and --blockvarpct; and K8 against K6 in their stage-in + verify forms
over PCIe. Old and new alternate within one process (CUDA events, warm-up launches, --reps
alternating runs); the card's name, power limit and max SM clock are read in the same run.

    python scripts/bench_dedupe.py [--window-gib 4] [--staged-gib 1] [--reps 3] [--out result.json]
"""
import argparse
import json
import os
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

from elbencho_b200 import kernels  # noqa: E402
from scripts.bench_verify_random import card_info, time_launches  # noqa: E402
from scripts.bench_verify_random_grain import SHAPES, descs_for, gbps  # noqa: E402

GiB, MiB, KiB = 1 << 30, 1 << 20, 1 << 10
SEED = 0xC0FFEE
GRAIN_SHIFTS = {"4KiB": 12, "64KiB": 16, "1MiB": 20}
DEDUPE_PCTS = [50, 100]


def resident(window, reps, pct):
    s = torch.cuda.current_stream().cuda_stream
    buf = torch.empty(window, dtype=torch.uint8, device="cuda")
    counters = torch.zeros(kernels.DEVCTR_NUM, dtype=torch.int64, device="cuda")
    out = {}
    for name, (block, hinting) in SHAPES.items():
        n = window // block
        hints = dict(total_bytes=window, max_block_len=block) if hinting == "hinted" else {}
        descs = descs_for(buf, window, block, True, "cuda")
        res = torch.empty(2 * n, dtype=torch.int64, device="cuda")
        init_ms = time_launches(lambda: kernels.verify_results_init(res.data_ptr(), n, s), 20)
        for g, shift in GRAIN_SHIFTS.items():
            runs = {"K5": [], "K6": []}
            runs.update({"K7_P%d" % p: [] for p in DEDUPE_PCTS})
            runs.update({"K8_P%d" % p: [] for p in DEDUPE_PCTS})
            for _ in range(reps):
                # (each verify run checks the content of the fill just before it)
                runs["K5"].append(time_launches(lambda: kernels.fill_random_grain_batch(
                    descs.data_ptr(), n, shift, pct, SEED, 0, s, **hints), 20))
                runs["K6"].append(time_launches(lambda: kernels.verify_random_grain_batch(
                    descs.data_ptr(), n, shift, pct, SEED, res.data_ptr(), counters.data_ptr(), s,
                    **hints), 20) - init_ms)
                assert int(counters[kernels.DEVCTR_VERIFY_MISMATCH_BYTES]) == 0
                for p in DEDUPE_PCTS:
                    runs["K7_P%d" % p].append(time_launches(lambda: kernels.fill_dedupe_grain_batch(
                        descs.data_ptr(), n, shift, pct, p, SEED, 0, s, **hints), 20))
                    runs["K8_P%d" % p].append(time_launches(
                        lambda: kernels.verify_dedupe_grain_batch(
                            descs.data_ptr(), n, shift, pct, p, SEED, res.data_ptr(),
                            counters.data_ptr(), s, **hints), 20) - init_ms)
                    assert int(counters[kernels.DEVCTR_VERIFY_MISMATCH_BYTES]) == 0
            cell = {k: dict(ms=[round(v, 4) for v in vals], gbps=gbps(window, vals))
                    for k, vals in runs.items()}
            for p in DEDUPE_PCTS:
                cell["K7_P%d_over_K5" % p] = round(min(runs["K5"]) / min(runs["K7_P%d" % p]), 3)
                cell["K8_P%d_over_K6" % p] = round(min(runs["K6"]) / min(runs["K8_P%d" % p]), 3)
            out["%s/G%s" % (name, g)] = cell
    del buf
    torch.cuda.empty_cache()
    return out


def staged(window, reps):
    """stage-in + verify over PCIe from pinned host memory, 1 MiB blocks, tiled shape, 64 KiB
    grains"""
    s = torch.cuda.current_stream().cuda_stream
    dev = torch.empty(window, dtype=torch.uint8, device="cuda")
    host = torch.empty(window, dtype=torch.uint8).pin_memory()
    delta = host.data_ptr() - dev.data_ptr()
    n = window // MiB
    hints = dict(total_bytes=window, max_block_len=MiB)
    descs = descs_for(dev, window, MiB, True, None)
    dev_res = torch.empty(2 * n, dtype=torch.int64, device="cuda")
    host_res = torch.empty(2 * n, dtype=torch.int64).pin_memory()
    ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
    kernels.verify_results_init(dev_res.data_ptr(), n, s)
    runs = {"K6": []}
    runs.update({"K8_P%d" % p: [] for p in DEDUPE_PCTS})
    for _ in range(reps):
        kernels.fill_random_grain_staged(descs.data_ptr(), n, 16, 100, SEED, delta, 0, s, **hints)
        runs["K6"].append(time_launches(lambda: kernels.verify_random_grain_staged(
            descs.data_ptr(), n, 16, 100, SEED, delta, dev_res.data_ptr(), host_res.data_ptr(),
            ticket.data_ptr(), 0, s, **hints), 5))
        assert all(v == 0 for v in host_res.tolist()[0::2])
        for p in DEDUPE_PCTS:
            kernels.fill_dedupe_grain_staged(descs.data_ptr(), n, 16, 100, p, SEED, delta, 0, s,
                                             **hints)
            runs["K8_P%d" % p].append(time_launches(lambda: kernels.verify_dedupe_grain_staged(
                descs.data_ptr(), n, 16, 100, p, SEED, delta, dev_res.data_ptr(),
                host_res.data_ptr(), ticket.data_ptr(), 0, s, **hints), 5))
            assert all(v == 0 for v in host_res.tolist()[0::2])
    return {k: dict(gib_per_s=[round(window / GiB / (v / 1e3), 2) for v in vals])
            for k, vals in runs.items()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--window-gib", type=float, default=4.0)
    p.add_argument("--staged-gib", type=float, default=1.0)
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--out", default=None)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dedupe.py needs a CUDA device")
    t0 = time.time()
    window = int(args.window_gib * GiB)
    result = dict(card=card_info(), window_gib=args.window_gib,
                  resident_pct100=resident(window, args.reps, 100),
                  resident_pct50=resident(window, args.reps, 50),
                  staged_tiled_1MiB_G64KiB=staged(int(args.staged_gib * GiB), args.reps))
    result["seconds"] = round(time.time() - t0, 1)
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
