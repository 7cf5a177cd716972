"""Times the measure pass against the decodes it serves, on device-resident batches (CUDA events).

    python tools/measure_bench.py [--blocks 131072] [--reps 5] [--classes E0,E50,E100,ETEXT] [--out FILE.json]

For each class: 2^17 x 64 KiB blocks are generated and encoded on the device (fast encoder) and compacted into one packed
payload; then each of these runs `--reps` times after a warm-up, and the mean time per call is reported:
  measure        lz4b200_measure_batch, unknown size, no capacities
  unknown        lz4b200_decode_batch, unknown size, exact capacities (64 KiB per block)
  packed         lz4b200_decode_batch_packed (measure + scan + decode)
  known          lz4b200_decode_batch, known size
Rates are decoded bytes over time.  Every call's results are checked (sizes = 64 KiB, the packed output equals the
known-size decode).  The card's name and power limit are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--blocks", type=int, default=1 << 17)
    p.add_argument("--reps", type=int, default=5)
    p.add_argument("--classes", default="E0,E50,E100,ETEXT")
    p.add_argument("--out", default=None)
    args = p.parse_args()

    import torch
    import lz4net_b200
    from lz4net_b200 import batch, synth
    if not torch.cuda.is_available():
        sys.exit("measure_bench.py needs a CUDA device")
    ctx = lz4net_b200.default_context()
    nb, bs = args.blocks, 65536
    slot = bs + bs // 255 + 16
    card, power = _card()
    results = {"card": card, "power_limit": power, "blocks": nb, "block_size": bs, "classes": {}}

    def timed(fn):
        fn()                                                        # warm-up
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.reps):
            fn()
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1) / args.reps

    for cls in args.classes.split(","):
        raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
        batch.synth_fill(ctx, raw, nb, bs, synth.CLASS_ID[cls], seed=5)
        so, do, sl, dc = batch.uniform_layout(nb, bs, slot, "cuda")
        slots = torch.empty(nb * slot, dtype=torch.uint8, device="cuda")
        clen = torch.zeros(nb, dtype=torch.int32, device="cuda")
        batch.encode(ctx, raw, so, sl, slots, do, dc, clen)
        coff = torch.zeros(nb + 1, dtype=torch.int64, device="cuda")
        comp = torch.empty(nb * slot, dtype=torch.uint8, device="cuda")
        batch.compact(ctx, slots, do, clen, comp, coff)
        del slots
        csrc = coff[:-1].contiguous()
        out = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
        size = torch.zeros(nb, dtype=torch.int32, device="cuda")
        res = torch.zeros(nb, dtype=torch.int32, device="cuda")
        out_off = torch.zeros(nb + 1, dtype=torch.int64, device="cuda")

        t = {
            "measure": timed(lambda: batch.measure(ctx, comp, csrc, clen, size)),
            "unknown": timed(lambda: batch.decode(ctx, comp, csrc, clen, out, so, sl, res, known=False)),
            "packed": timed(lambda: batch.decode_packed(ctx, comp, csrc, clen, out, out_off, res)),
            "known": timed(lambda: batch.decode(ctx, comp, csrc, clen, out, so, sl, res, known=True)),
        }
        torch.cuda.synchronize()
        assert bool((size == bs).all()) and bool((res == clen).all()), cls
        assert torch.equal(out, raw), cls
        del raw
        ratio = float(clen.sum()) / (nb * bs)
        row = {"ratio": round(ratio, 4)}
        for k, ms in t.items():
            row[k + "_ms"] = round(ms, 3)
            row[k + "_gbs"] = round(nb * bs / ms / 1e6, 1)
        row["measure_over_unknown"] = round(t["measure"] / t["unknown"], 3)
        results["classes"][cls] = row
        print(cls, json.dumps(row), flush=True)
        del comp, out
        torch.cuda.empty_cache()
    print(json.dumps(results))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
