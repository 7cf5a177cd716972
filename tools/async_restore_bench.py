"""Measures the offload -> restore round trip with the restore taking the offsets the offload wrote on the device
(lz4b200_decode_batch_to_device_at_async, lz4b200_unwrap_batch_to_device_at_async), against the way without them:
synchronise, read out_off on the host, then lz4b200_decode_batch_to_device_async / unwrap_batch_to_device_async.

    python tools/async_restore_bench.py [--blocks 16384] [--block-size 65536] [--reps 5] [--classes E0,E50,ETEXT]
                                        [--host-chunk-mb MB] [--out FILE.json]

Per class (E0, E50, ETEXT), with the card's name and power limit read in the same run:
  round    wall time (host clock around both calls + a synchronise) and host time until the restore call has returned,
           for the codec (asynchronous packed encode, then decode) and for Wrap packets (asynchronous packed Wrap, then
           Unwrap); median of --reps after one warm-up.  The restored bytes and out_len are checked every time.
  staging  (E0 only) the lift kernel's rate in GB/s of bytes staged, from its torch.profiler device time over one restore
           (the codec's), beside a cudaMemcpyAsync H2D of the same number of bytes from page-locked memory, timed with
           CUDA events.
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
    try:
        q = "power.limit,clocks.max.sm,pcie.link.gen.current,pcie.link.width.current"
        info = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        info = "unknown"
    return torch.cuda.get_device_name(0), info


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--blocks", type=int, default=1 << 14)
    p.add_argument("--block-size", type=int, default=65536)
    p.add_argument("--reps", type=int, default=5)
    p.add_argument("--classes", default="E0,E50,ETEXT")
    p.add_argument("--host-chunk-mb", type=int, default=0, help="pipeline stage size (0: the library's default)")
    p.add_argument("--out", default=None)
    args = p.parse_args()

    import numpy as np
    import torch
    import lz4net_b200
    from lz4net_b200 import batch, synth
    if not torch.cuda.is_available():
        sys.exit("async_restore_bench.py needs a CUDA device")
    card, info = _card()
    res = {"card": card, "power_limit,max_sm_clock,pcie_gen,pcie_width": info, "blocks": args.blocks,
           "block_size": args.block_size, "reps": args.reps, "host_chunk_mb": args.host_chunk_mb or "default", "classes": []}
    print(json.dumps({k: res[k] for k in ("card", "power_limit,max_sm_clock,pcie_gen,pcie_width")}), flush=True)
    ctx = lz4net_b200.default_context()
    if args.host_chunk_mb:
        ctx.set_option("host_chunk_mb", args.host_chunk_mb)
    n, bs = args.blocks, args.block_size
    raw = torch.empty(n * bs, dtype=torch.uint8, device="cuda")
    back = torch.empty_like(raw)
    so = np.arange(n, dtype=np.int64) * bs
    sl = np.full(n, bs, np.int32)
    bound = np.full(n, bs + bs // 255 + 16, np.int32)
    caps = {"codec": int(bound.sum()), "wrap": n * (bs + 8)}
    host = {k: torch.empty(v, dtype=torch.uint8).pin_memory() for k, v in caps.items()}
    off, out_len = torch.empty(n + 1, dtype=torch.int64, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda")
    r_len = torch.empty(n, dtype=torch.int32, device="cuda")

    def offload(kind):
        if kind == "codec":
            batch.encode_to_host_packed_async(ctx, raw, so, sl, bound, host[kind], off, out_len)
        else:
            batch.wrap_to_host_packed_async(ctx, raw, so, sl, host[kind], off, out_len)

    def restore_at(kind):
        if kind == "codec":
            batch.decode_from_host_at_async(ctx, host[kind], caps[kind], off, back, so, sl, r_len)
        else:
            batch.unwrap_to_device_at_async(ctx, host[kind], caps[kind], off, back, so, sl, r_len)

    def restore_host(kind):
        torch.cuda.current_stream().synchronize()
        o = off.cpu().numpy()
        hs, hl = o[:n].copy(), np.diff(o).astype(np.int32)
        if kind == "codec":
            batch.decode_from_host_async(ctx, host[kind], hs, hl, back, so, sl, r_len)
        else:
            batch.unwrap_to_device_async(ctx, host[kind], hs, hl, back, so, sl, r_len)

    for cls in args.classes.split(","):
        batch.synth_fill(ctx, raw, n, bs, synth.CLASS_ID[cls])
        torch.cuda.synchronize()
        row = {"class": cls, "raw_bytes": n * bs}
        for kind in ("codec", "wrap"):
            times = {"device_offsets": [], "host_offsets": []}
            for rep in range(args.reps + 1):
                for path, restore in (("device_offsets", restore_at), ("host_offsets", restore_host)):
                    back.zero_()
                    r_len.fill_(12345)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    offload(kind)
                    restore(kind)
                    inside = time.perf_counter() - t0
                    torch.cuda.synchronize()
                    wall = time.perf_counter() - t0
                    # a known-size decode reports the bytes it read, an Unwrap the bytes it restored
                    want_len = torch.diff(off) if kind == "codec" else torch.full_like(off[1:], bs)
                    assert torch.equal(r_len.long(), want_len) and torch.equal(back, raw), (cls, kind, path)
                    if rep:
                        times[path].append({"wall_ms": wall * 1e3, "in_call_ms": inside * 1e3})
            row[kind] = {"host_bytes": int(off[-1].item())}
            for path, v in times.items():
                row[kind][path] = {"wall_ms_median": float(np.median([x["wall_ms"] for x in v])),
                                   "wall_ms_min": min(x["wall_ms"] for x in v),
                                   "in_call_ms_median": float(np.median([x["in_call_ms"] for x in v]))}
        if cls == "E0":
            row["staging"] = staging(ctx, n, offload, restore_at, off)
        res["classes"].append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


def staging(ctx, n, offload, restore_at, off):
    """The lift kernel's device time over one codec restore (torch.profiler), and an H2D copy of as many bytes."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    offload("codec")
    torch.cuda.synchronize()
    staged = int(off[-1].item())                                          # the spans' bytes: what the kernel stages
    restore_at("codec")                                                   # warm
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        restore_at("codec")
        torch.cuda.synchronize()
    lift_us, launches = 0.0, 0
    for e in prof.events():
        if "lz4_lift_kernel" in e.name and e.device_type == torch.autograd.DeviceType.CUDA:
            lift_us += e.time_range.elapsed_us()
            launches += 1
    src = torch.empty(staged, dtype=torch.uint8).pin_memory()
    dst = torch.empty(staged, dtype=torch.uint8, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    copies = []
    for rep in range(6):
        ev[0].record()
        dst.copy_(src, non_blocking=True)
        ev[1].record()
        torch.cuda.synchronize()
        if rep:
            copies.append(ev[0].elapsed_time(ev[1]))
    copy_ms = sorted(copies)[len(copies) // 2]
    return {"staged_bytes": staged, "lift_launches": launches, "lift_ms": lift_us / 1e3,
            "lift_GBps": staged / (lift_us * 1e3) if lift_us else None,
            "h2d_copy_ms_median": copy_ms, "h2d_copy_GBps": staged / (copy_ms * 1e6)}


if __name__ == "__main__":
    main()
