"""Measures the LZ4Stream round trip with no host wait (lz4b200_stream_encode_from_device_async, then
lz4b200_stream_decode_to_device_at_async, which reads the stream's size and walks its headers on the device) against the
round trip that has to wait for the size (the same encode, a synchronise, then lz4b200_stream_decode_to_device_async,
which walks the headers on the host).

    python tools/async_stream_restore_bench.py [--mib 1024] [--hc-mib 64] [--reps 3] [--out FILE.json]

Per class (E0, E50, E100, ETEXT) and chunk size (64 KiB, 1 MiB), fast mode on --mib MiB and HC on --hc-mib MiB, with the
card's name, power limit and PCIe link read in the same run:
  wait / at      end to end: device events around the whole round trip, and the host clock to the final synchronise;
                 the host time until each call returned (the wait form's includes its synchronise on the encode)
  walk_ms        the device walk kernels' total time in one round trip (torch.profiler, a separate run; kernel
                 lz4_stream_walk_kernel)
Every restored tensor is compared with the source, and out_size with its length.
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
    p.add_argument("--mib", type=int, default=1024)
    p.add_argument("--hc-mib", type=int, default=64)
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--out", default=None)
    args = p.parse_args()

    import numpy as np
    import torch
    import lz4net_b200
    from lz4net_b200 import batch, native, synth
    if not torch.cuda.is_available():
        sys.exit("async_stream_restore_bench.py needs a CUDA device")
    card, info = _card()
    res = {"card": card, "power_limit,max_sm_clock,pcie_gen,pcie_width": info, "mib": args.mib, "hc_mib": args.hc_mib,
           "reps": args.reps, "rows": []}
    print(json.dumps({k: res[k] for k in ("card", "power_limit,max_sm_clock,pcie_gen,pcie_width")}), flush=True)
    ctx = lz4net_b200.default_context()
    lib = native.lib()
    fill_bs = 65536
    n_max = args.mib << 20
    raw_all = torch.empty(n_max, dtype=torch.uint8, device="cuda")
    back_all = torch.empty_like(raw_all)
    wire = torch.empty(int(lib.lz4b200_stream_bound(n_max, fill_bs)), dtype=torch.uint8).pin_memory()
    size = torch.empty(1, dtype=torch.int64, device="cuda")
    out = torch.empty(1, dtype=torch.int64, device="cuda")
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def wait_form(raw, back, bs, hc, cap):
        t0 = time.perf_counter()
        batch.stream_encode_to_host_async(ctx, raw, wire[:cap], size, block_size=bs, hc=hc)
        t1 = time.perf_counter()
        n = int(size.item())                                            # the host wait this form cannot avoid
        batch.stream_decode_to_device_async(ctx, wire, n, back, out)
        return t1 - t0, time.perf_counter() - t1

    def at_form(raw, back, bs, hc, cap):
        t0 = time.perf_counter()
        batch.stream_encode_to_host_async(ctx, raw, wire[:cap], size, block_size=bs, hc=hc)
        t1 = time.perf_counter()
        batch.stream_decode_to_device_at_async(ctx, wire, cap, size, back, out, block_size=bs)
        return t1 - t0, time.perf_counter() - t1

    for hc, mib in ((False, args.mib), (True, args.hc_mib)):
        n = mib << 20
        raw, back = raw_all[:n], back_all[:n]
        for cls in ("E0", "E50", "E100", "ETEXT"):
            batch.synth_fill(ctx, raw, n // fill_bs, fill_bs, synth.CLASS_ID[cls])
            torch.cuda.synchronize()
            for bs in (65536, 1 << 20):
                cap = int(lib.lz4b200_stream_bound(n, bs))
                row = {"class": cls, "mode": "hc" if hc else "fast", "block_size": bs, "raw_bytes": n, "outputs_equal": True}
                for name, form in (("wait", wait_form), ("at", at_form)):
                    v = []
                    for rep in range(args.reps + 1):
                        back.zero_()
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        ev0.record()
                        enc_s, dec_s = form(raw, back, bs, hc, cap)
                        ev1.record()
                        torch.cuda.synchronize()
                        wall = time.perf_counter() - t0
                        ok = int(out.item()) == n and torch.equal(back, raw)
                        row["outputs_equal"] &= ok
                        if rep:
                            v.append((ev0.elapsed_time(ev1), wall * 1e3, enc_s * 1e3, dec_s * 1e3))
                    a = np.array(v)
                    row[name] = {"device_ms_median": float(np.median(a[:, 0])), "wall_ms_median": float(np.median(a[:, 1])),
                                 "encode_return_ms_median": float(np.median(a[:, 2])),
                                 "decode_return_ms_median": float(np.median(a[:, 3]))}
                row["stream_bytes"] = int(size.item())
                row["at_over_wait_wall"] = row["at"]["wall_ms_median"] / row["wait"]["wall_ms_median"]
                # the walk's cost, in a run of its own
                torch.cuda.synchronize()
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    at_form(raw, back, bs, hc, cap)
                    torch.cuda.synchronize()
                walks = [e for e in prof.events() if "lz4_stream_walk_kernel" in e.name]
                row["walk_ms"] = sum(e.device_time_total for e in walks) / 1e3
                row["walk_launches"] = len(walks)
                row["outputs_equal"] &= int(out.item()) == n and torch.equal(back, raw)
                res["rows"].append(row)
                print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
