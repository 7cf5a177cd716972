"""Measures the asynchronous Wrap into page-locked host memory and the asynchronous packed Unwrap back
(lz4b200_wrap_batch_packed_from_device_async, lz4b200_unwrap_batch_packed_to_device_async) against their synchronous
forms, and what the packets cost in host memory against the bare blocks of the asynchronous packed encode.

    python tools/async_wrap_bench.py [--blocks 16384] [--block-size 65536] [--reps 5] [--out FILE.json]

Per class (E0, E50, E100, ETEXT), with the card's name, power limit and PCIe link read in the same run:
  calls    wall time (host clock around call + synchronise) and host time inside the call, synchronous against
           asynchronous, for the packed Wrap (device -> page-locked host) and the packed Unwrap (page-locked host -> device).
  bytes    host bytes per raw byte: the packets, against lz4b200_encode_batch_packed_from_device_async at
           dst_cap = MaximumOutputLength(len); and how many blocks that encode fails at dst_cap = len.
Every output is compared with the synchronous call's (the Wrap's offsets, lengths and bytes; the Unwrap's offsets,
lengths and restored bytes, which must equal the source).
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
        sys.exit("async_wrap_bench.py needs a CUDA device")
    card, info = _card()
    res = {"card": card, "power_limit,max_sm_clock,pcie_gen,pcie_width": info, "blocks": args.blocks,
           "block_size": args.block_size, "reps": args.reps, "classes": []}
    print(json.dumps({k: res[k] for k in ("card", "power_limit,max_sm_clock,pcie_gen,pcie_width")}), flush=True)
    ctx = lz4net_b200.default_context()
    n, bs = args.blocks, args.block_size
    raw = torch.empty(n * bs, dtype=torch.uint8, device="cuda")
    back = torch.empty_like(raw)
    so = np.arange(n, dtype=np.int64) * bs
    sl = np.full(n, bs, np.int32)
    bound = np.full(n, bs + bs // 255 + 16, np.int32)
    wire = torch.empty(n * (bs + 8), dtype=torch.uint8).pin_memory()          # sum(len + 8): always enough
    host = wire.numpy()
    blocks_dst = torch.empty(int(bound.sum()), dtype=torch.uint8).pin_memory()
    off, out_len = torch.empty(n + 1, dtype=torch.int64, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda")
    u_off, u_len = torch.empty(n + 1, dtype=torch.int64, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda")

    for cls in ("E0", "E50", "E100", "ETEXT"):
        batch.synth_fill(ctx, raw, n, bs, synth.CLASS_ID[cls])
        torch.cuda.synchronize()
        w_off, w_len = np.zeros(n + 1, np.int64), np.zeros(n, np.int32)
        total = batch.wrap_to_host_packed(ctx, raw, so, sl, host, w_off, w_len)
        want = host[:total].copy()
        p_off, p_len = w_off[:n].copy(), w_len.copy()
        r_off, r_len = np.zeros(n + 1, np.int64), np.zeros(n, np.int32)
        want_u_off = np.arange(n + 1, dtype=np.int64) * bs

        def check(path):
            if path == "wrap_sync":
                assert np.array_equal(w_off, np.concatenate([[0], np.cumsum(p_len)])) and np.array_equal(w_len, p_len), path
                assert np.array_equal(host[:total], want), path
            elif path == "wrap_async":
                assert np.array_equal(off.cpu().numpy(), w_off) and np.array_equal(out_len.cpu().numpy(), p_len), path
                assert np.array_equal(host[:total], want), path
            else:
                got_off, got_len = (r_off, r_len) if path == "unwrap_sync" else (u_off.cpu().numpy(), u_len.cpu().numpy())
                assert np.array_equal(got_off, want_u_off) and (got_len == bs).all(), path
                assert torch.equal(back, raw), path
                back.zero_()

        rows = {"wrap_sync": [], "wrap_async": [], "unwrap_sync": [], "unwrap_async": []}
        for rep in range(args.reps + 1):
            for path in rows:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if path == "wrap_sync":
                    batch.wrap_to_host_packed(ctx, raw, so, sl, host, w_off, w_len)
                elif path == "wrap_async":
                    batch.wrap_to_host_packed_async(ctx, raw, so, sl, wire, off, out_len)
                elif path == "unwrap_sync":
                    batch.unwrap_to_device_packed(ctx, host, p_off, p_len, back, r_off, r_len)
                else:
                    batch.unwrap_to_device_packed_async(ctx, wire, p_off, p_len, back, u_off, u_len)
                inside = time.perf_counter() - t0
                torch.cuda.synchronize()
                wall = time.perf_counter() - t0
                check(path)
                if rep:
                    rows[path].append({"wall_ms": wall * 1e3, "in_call_ms": inside * 1e3})
        # host bytes: the packets against the bare blocks of the asynchronous packed encode at the bound, and how many
        # blocks that encode fails at a capacity of their own length
        batch.encode_to_host_packed_async(ctx, raw, so, sl, bound, blocks_dst, off, out_len)
        torch.cuda.synchronize()
        blocks_total = int(off[-1].item())
        batch.encode_to_host_packed_async(ctx, raw, so, sl, sl, blocks_dst, off, out_len)
        torch.cuda.synchronize()
        failed_at_len = int((out_len == 0).sum().item())
        row = {"class": cls, "raw_bytes": n * bs, "packet_bytes": int(total), "packets_per_raw": total / (n * bs),
               "blocks_at_bound_bytes": blocks_total, "blocks_at_bound_per_raw": blocks_total / (n * bs),
               "blocks_failed_at_cap_len": failed_at_len, "stored_raw_packets": int((p_len == bs + 8).sum())}
        for path, v in rows.items():
            row[path] = {"wall_ms_min": min(x["wall_ms"] for x in v), "wall_ms_median": float(np.median([x["wall_ms"] for x in v])),
                         "in_call_ms_median": float(np.median([x["in_call_ms"] for x in v]))}
        res["classes"].append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
