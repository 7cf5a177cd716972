"""Measures the asynchronous offload calls (lz4b200_encode_batch_packed_from_device_async,
lz4b200_decode_batch_to_device_async) on the GPU.

    python tools/async_offload_bench.py [--blocks 16384] [--block-size 65536] [--reps 5] [--out FILE.json]

Three parts, with the card's name, power limit and PCIe link read in the same run:
  land     the landing kernel's host-write rate (its bytes over its kernel time, from torch.profiler, in an async encode
           of incompressible E0 blocks), against cudaMemcpyAsync device -> page-locked host of the same bytes (CUDA events).
  calls    the async against the synchronous packed encode (device -> page-locked host) and known-size decode (page-locked
           host -> device) on E50 and ETEXT: wall time (host clock around call + synchronise) and host time inside the call.
  overlap  the async encode beside a compute-bound kernel (bf16 matmuls) on another stream, against the two run alone.
Every output is checked against the source (decode) or the synchronous call (encode).
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
    p.add_argument("--out", default=None)
    args = p.parse_args()

    import numpy as np
    import torch
    import lz4net_b200
    from lz4net_b200 import batch, synth
    if not torch.cuda.is_available():
        sys.exit("async_offload_bench.py needs a CUDA device")
    card, info = _card()
    res = {"card": card, "power_limit,max_sm_clock,pcie_gen,pcie_width": info, "blocks": args.blocks,
           "block_size": args.block_size, "reps": args.reps}
    print(json.dumps({k: res[k] for k in ("card", "power_limit,max_sm_clock,pcie_gen,pcie_width")}), flush=True)
    ctx = lz4net_b200.default_context()
    n, bs = args.blocks, args.block_size
    raw = torch.empty(n * bs, dtype=torch.uint8, device="cuda")
    so = np.arange(n, dtype=np.int64) * bs
    sl = np.full(n, bs, np.int32)
    caps = np.full(n, bs + bs // 255 + 16, np.int32)
    dst = torch.empty(int(caps.sum()), dtype=torch.uint8).pin_memory()
    off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    out_len = torch.empty(n, dtype=torch.int32, device="cuda")

    def fill(cls):
        batch.synth_fill(ctx, raw, n, bs, synth.CLASS_ID[cls])
        torch.cuda.synchronize()

    def enc_async(stream=None):
        t0 = time.perf_counter()
        batch.encode_to_host_packed_async(ctx, raw, so, sl, caps, dst, off, out_len, stream=stream)
        return time.perf_counter() - t0

    # ---- land: kernel host-write rate against a copy-engine D2H of the same bytes ----
    fill("E0")
    enc_async(); torch.cuda.synchronize()
    total = int(off[-1].item())
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        enc_async(); torch.cuda.synchronize()
    land_us = sum(e.device_time_total for e in prof.key_averages() if "lz4_land_kernel" in e.key)
    land_calls = sum(e.count for e in prof.key_averages() if "lz4_land_kernel" in e.key)
    dev_copy = torch.empty(total, dtype=torch.uint8, device="cuda")
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(args.reps):
        a.record(); dst[:total].copy_(dev_copy, non_blocking=True); b.record(); torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    res["land"] = {"bytes": total, "land_kernel_us": land_us, "land_kernels": land_calls,
                   "land_GBps": total / (land_us * 1e3) if land_us else None,
                   "memcpy_d2h_ms": ms, "memcpy_d2h_GBps": total / (min(ms) * 1e6)}
    print(json.dumps({"land": res["land"]}), flush=True)

    # ---- calls: async against sync, encode and decode ----
    res["calls"] = []
    host = dst.numpy()
    for cls in ("E50", "ETEXT"):
        fill(cls)
        src_bytes = raw.cpu().numpy()
        w_off, w_len = np.zeros(n + 1, np.int64), np.zeros(n, np.int32)
        batch.encode_to_host_packed(ctx, raw, so, sl, caps, host, w_off, w_len)
        want = host[:w_off[-1]].tobytes()
        comp_off, comp_len = w_off[:n].copy(), w_len.copy()
        back = torch.empty(n * bs, dtype=torch.uint8, device="cuda")
        d_len = np.zeros(n, np.int32)
        d_len_t = torch.empty(n, dtype=torch.int32, device="cuda")
        rows = {"encode_sync": [], "encode_async": [], "decode_sync": [], "decode_async": []}
        for rep in range(args.reps + 1):
            for path in rows:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if path == "encode_sync":
                    batch.encode_to_host_packed(ctx, raw, so, sl, caps, host, w_off, w_len); inside = time.perf_counter() - t0
                elif path == "encode_async":
                    inside = enc_async()
                elif path == "decode_sync":
                    batch.decode_from_host(ctx, host, comp_off, comp_len, back, so, sl, d_len); inside = time.perf_counter() - t0
                else:
                    batch.decode_from_host_async(ctx, dst, comp_off, comp_len, back, so, sl, d_len_t)
                    inside = time.perf_counter() - t0
                torch.cuda.synchronize()
                wall = time.perf_counter() - t0
                if path.startswith("encode"):
                    assert host[:int(off[-1].item()) if path == "encode_async" else w_off[-1]].tobytes() == want, path
                else:
                    assert back.cpu().numpy().tobytes() == src_bytes.tobytes(), path
                    back.zero_()
                if rep:
                    rows[path].append({"wall_ms": wall * 1e3, "in_call_ms": inside * 1e3})
        row = {"class": cls, "raw_bytes": n * bs, "compressed_bytes": len(want)}
        for path, v in rows.items():
            row[path] = {"wall_ms_min": min(x["wall_ms"] for x in v), "wall_ms_median": float(np.median([x["wall_ms"] for x in v])),
                         "in_call_ms_median": float(np.median([x["in_call_ms"] for x in v]))}
        res["calls"].append(row)
        print(json.dumps(row), flush=True)

    # ---- overlap: the async encode beside a compute-bound kernel on another stream ----
    fill("E50")
    x = torch.randn(8192, 8192, device="cuda", dtype=torch.bfloat16)
    y = torch.empty_like(x)
    compute, codec = torch.cuda.Stream(), torch.cuda.Stream()
    iters = 40

    def run(do_compute, do_encode):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if do_compute:
            with torch.cuda.stream(compute):
                for _ in range(iters):
                    torch.matmul(x, x, out=y)
        if do_encode:
            enc_async(codec)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    run(True, True)
    ov = {"compute_alone_ms": [], "encode_alone_ms": [], "both_ms": []}
    for _ in range(args.reps):
        ov["compute_alone_ms"].append(run(True, False))
        ov["encode_alone_ms"].append(run(False, True))
        ov["both_ms"].append(run(True, True))
    ov = {k: float(np.median(v)) for k, v in ov.items()}
    ov["matmuls"] = f"{iters} x bf16 8192^3"
    res["overlap"] = ov
    print(json.dumps({"overlap": ov}), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
