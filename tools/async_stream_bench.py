"""Measures the asynchronous LZ4Stream encode into page-locked host memory and the asynchronous decode back
(lz4b200_stream_encode_from_device_async, lz4b200_stream_decode_to_device_async) against their synchronous forms
(lz4b200_stream_encode_from_device, lz4b200_stream_decode_to_device into the same page-locked buffers).

    python tools/async_stream_bench.py [--mib 1024] [--hc-mib 64] [--reps 3] [--out FILE.json]

Per class (E0, E50, E100, ETEXT) and chunk size (64 KiB, 1 MiB), fast mode on --mib MiB and HC on --hc-mib MiB, with the
card's name, power limit and PCIe link read in the same run:
  encode / decode   wall time (host clock around call + synchronise) and host time inside the call, synchronous against
                    asynchronous, and the stream's size per raw byte.
Every output is compared with the synchronous call's: the encode's size and bytes, the decode's size and restored bytes,
which must equal the source.
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


def _stats(v):
    import numpy as np
    return {"wall_ms_min": min(x["wall_ms"] for x in v), "wall_ms_median": float(np.median([x["wall_ms"] for x in v])),
            "in_call_ms_median": float(np.median([x["in_call_ms"] for x in v]))}


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
        sys.exit("async_stream_bench.py needs a CUDA device")
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
    cap_max = int(lib.lz4b200_stream_bound(n_max, fill_bs))
    wire_sync = torch.empty(cap_max, dtype=torch.uint8).pin_memory()
    wire_async = torch.empty(cap_max, dtype=torch.uint8).pin_memory()
    size = torch.empty(1, dtype=torch.int64, device="cuda")
    dsize = torch.empty(1, dtype=torch.int64, device="cuda")

    for hc, mib in ((False, args.mib), (True, args.hc_mib)):
        n = mib << 20
        raw, back = raw_all[:n], back_all[:n]
        for cls in ("E0", "E50", "E100", "ETEXT"):
            batch.synth_fill(ctx, raw, n // fill_bs, fill_bs, synth.CLASS_ID[cls])
            torch.cuda.synchronize()
            for bs in (65536, 1 << 20):
                cap = int(lib.lz4b200_stream_bound(n, bs))
                ws, wa = wire_sync[:cap], wire_async[:cap]
                want = batch.stream_encode_to_host(ctx, raw, block_size=bs, hc=hc, dst=ws.numpy())
                w = len(want)
                want_copy = want.copy()
                rows = {"encode_sync": [], "encode_async": [], "decode_sync": [], "decode_async": []}
                for rep in range(args.reps + 1):
                    for path in rows:
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        if path == "encode_sync":
                            got = len(batch.stream_encode_to_host(ctx, raw, block_size=bs, hc=hc, dst=ws.numpy()))
                        elif path == "encode_async":
                            batch.stream_encode_to_host_async(ctx, raw, wa, size, block_size=bs, hc=hc)
                        elif path == "decode_sync":
                            got = batch.stream_decode_to_device(ctx, ws.numpy()[:w], back)
                        else:
                            batch.stream_decode_to_device_async(ctx, wa, w, back, dsize)
                        inside = time.perf_counter() - t0
                        torch.cuda.synchronize()
                        wall = time.perf_counter() - t0
                        if path == "encode_sync":
                            assert got == w and np.array_equal(ws.numpy()[:w], want_copy), path
                        elif path == "encode_async":
                            assert int(size.item()) == w and np.array_equal(wa.numpy()[:w], want_copy), path
                        else:
                            got = got if path == "decode_sync" else int(dsize.item())
                            assert got == n and torch.equal(back, raw), path
                            back.zero_()
                        if rep:
                            rows[path].append({"wall_ms": wall * 1e3, "in_call_ms": inside * 1e3})
                row = {"class": cls, "mode": "hc" if hc else "fast", "block_size": bs, "raw_bytes": n, "stream_bytes": w,
                       "stream_per_raw": w / n, "outputs_equal": True}
                row.update({path: _stats(v) for path, v in rows.items()})
                for op in ("encode", "decode"):
                    row[f"{op}_async_over_sync_wall"] = row[f"{op}_async"]["wall_ms_median"] / row[f"{op}_sync"]["wall_ms_median"]
                res["rows"].append(row)
                print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
