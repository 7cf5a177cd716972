"""Times device-memory calls enqueued eagerly against the same calls replayed from a CUDA graph (host clock).

    python tools/graph_bench.py [--reps 200] [--warmup 20] [--blocks 32,256,2048] [--sizes 4096,65536] [--out FILE.json]

For every block count and block size, E50 blocks are generated on the device, and each workload below runs --reps times
after --warmup runs, each run ending in a torch.cuda.synchronize(); the host clock around the whole loop over --reps is
the per-call time reported:
  encode   lz4b200_encode_batch(MEM_DEVICE), fast
  decode   lz4b200_decode_batch(MEM_DEVICE), known size, of the blocks encode made
  chain    encode -> lz4b200_compact -> lz4b200_decode_batch_packed
"eager" enqueues the calls through the Python helpers (ctypes, the context's lock, the device switch, the launches);
"graph" replays a graph captured from the same helpers on a context that reserved the scratch first.  Both give the same
bytes, which is checked (same_bytes), as is the round trip.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def _timed(fn, reps, warmup):
    import torch
    for _ in range(warmup):
        fn()
        torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
        torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--blocks", default="32,256,2048")
    p.add_argument("--sizes", default="4096,65536")
    p.add_argument("--workloads", default="encode,decode,chain")
    p.add_argument("--out", default=None)
    args = p.parse_args()

    import torch
    from lz4net_b200 import batch
    from lz4net_b200.codec import Context
    if not torch.cuda.is_available():
        sys.exit("graph_bench.py needs a CUDA device")
    card, power = _card()
    results = {"card": card, "power_limit_and_max_sm_clock": power, "class": "E50", "reps": args.reps, "runs": []}
    ctx = Context(0)
    for nb in (int(x) for x in args.blocks.split(",")):
        for bs in (int(x) for x in args.sizes.split(",")):
            slot = bs + bs // 255 + 16
            dev = "cuda"
            raw = torch.empty(nb * bs, dtype=torch.uint8, device=dev)
            batch.synth_fill(ctx, raw, nb, bs, 1, seed=7)
            so, do, sl, dc = batch.uniform_layout(nb, bs, slot, dev)
            ro, _, rl, rc = batch.uniform_layout(nb, bs, bs, dev)
            t = dict(slots=torch.zeros(nb * slot, dtype=torch.uint8, device=dev), out=torch.zeros(nb, dtype=torch.int32, device=dev),
                     back=torch.zeros(nb * bs, dtype=torch.uint8, device=dev), bout=torch.zeros(nb, dtype=torch.int32, device=dev),
                     packed=torch.zeros(nb * slot, dtype=torch.uint8, device=dev), off=torch.zeros(nb + 1, dtype=torch.int64, device=dev),
                     pback=torch.zeros(nb * bs, dtype=torch.uint8, device=dev), poff=torch.zeros(nb + 1, dtype=torch.int64, device=dev),
                     pout=torch.zeros(nb, dtype=torch.int32, device=dev))
            work = {
                "encode": lambda: batch.encode(ctx, raw, so, sl, t["slots"], do, dc, t["out"]),
                "decode": lambda: batch.decode(ctx, t["slots"], do, t["out"], t["back"], ro, rc, t["bout"]),
                "chain": lambda: (batch.encode(ctx, raw, so, sl, t["slots"], do, dc, t["out"]),
                                  batch.compact(ctx, t["slots"], do, t["out"], t["packed"], t["off"]),
                                  batch.decode_packed(ctx, t["packed"], t["off"][:nb], t["out"], t["pback"], t["poff"], t["pout"])),
            }
            ctx.reserve(nb)
            work["encode"]()
            torch.cuda.synchronize()
            for name, fn in ((k, work[k]) for k in args.workloads.split(",")):
                eager = _timed(fn, args.reps, args.warmup)
                want = {k: v.clone() for k, v in t.items()}
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    fn()
                graph = _timed(g.replay, args.reps, args.warmup)
                same = all(torch.equal(t[k], want[k]) for k in t)
                del g
                row = {"workload": name, "blocks": nb, "block_size": bs, "eager_us": round(eager * 1e6, 2),
                       "graph_us": round(graph * 1e6, 2), "saved_us": round((eager - graph) * 1e6, 2), "same_bytes": same}
                print(json.dumps(row), flush=True)
                results["runs"].append(row)
            for name, out in (("decode", "back"), ("chain", "pback")):
                if name in args.workloads.split(",") and not torch.equal(t[out], raw):
                    print(json.dumps({"workload": name, "blocks": nb, "block_size": bs, "round_trip": False}), flush=True)
    ctx.close()
    print(json.dumps({k: results[k] for k in ("card", "power_limit_and_max_sm_clock")}), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
