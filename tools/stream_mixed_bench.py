"""Times the LZ4Stream calls between device and host memory against the workarounds they replace (host clock around
synchronous work).

    python tools/stream_mixed_bench.py [--gib 2] [--reps 2] [--classes E0,E50,E100,ETEXT] [--out FILE.json]

For each class, --gib GiB of raw data are generated in HBM; every host buffer is page-locked.  Configurations: 64 KiB and
1 MiB blocks with the fast encoder, and 1 MiB blocks with HC on E50 and ETEXT.  Paths, library defaults:
  encode_new         lz4b200_stream_encode_from_device: device raw -> stream bytes in host memory
  encode_workaround  one D2H copy of the raw bytes + lz4b200_stream_encode (host -> host)
  decode_new         lz4b200_stream_decode_to_device: host stream bytes -> device raw
  decode_workaround  lz4b200_stream_decode (host -> host) + one H2D copy of the raw bytes
Each path runs once on a fresh context (its device-memory high-water mark is read there: free memory before the first
call minus free memory after it, device-wide, with the path's buffers held; the raw data and the decode's output tensor
are allocated before and not counted), then --reps times; the mean time per call is reported.  Rates are raw bytes over
time.  The new and workaround streams are asserted byte-equal, and both decodes equal to the raw data, in the same run.
The card's name, power limit, max SM clock and PCIe link are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from mixed_memory_bench import _card  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--gib", type=float, default=2.0)
    p.add_argument("--reps", type=int, default=2)
    p.add_argument("--classes", default="E0,E50,E100,ETEXT")
    p.add_argument("--out", default=None)
    args = p.parse_args()

    import numpy as np
    import torch
    import lz4net_b200
    from lz4net_b200 import batch, native, synth
    if not torch.cuda.is_available():
        sys.exit("stream_mixed_bench.py needs a CUDA device")
    l = native.lib()
    synth_bs = 1 << 20
    nraw = int(args.gib * (1 << 30)) // synth_bs * synth_bs
    card, info = _card()
    results = {"card": card, "power_limit,max_sm_clock,pcie_gen,pcie_width": info, "raw_bytes": nraw,
               "device_hwm": "device-wide, torch.cuda.mem_get_info", "classes": {}}
    cap = int(l.lz4b200_stream_bound(nraw, 1 << 16))
    wire_new = torch.empty(cap, dtype=torch.uint8).pin_memory().numpy()
    wire_wa = torch.empty(cap, dtype=torch.uint8).pin_memory().numpy()
    hraw = torch.empty(nraw, dtype=torch.uint8).pin_memory()

    def run(setup, fn):
        """setup(ctx) -> state (allocates what the path holds); fn(ctx, state) runs one call and synchronises."""
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free0 = torch.cuda.mem_get_info()[0]
        ctx = lz4net_b200.Context(0)
        state = setup(ctx)
        fn(ctx, state)
        torch.cuda.synchronize()
        hwm = free0 - torch.cuda.mem_get_info()[0]
        t = time.perf_counter()
        for _ in range(args.reps):
            fn(ctx, state)
        ms = (time.perf_counter() - t) * 1e3 / args.reps
        ctx.close()
        return {"ms": round(ms, 2), "raw_gbs": round(nraw / ms / 1e6, 2), "device_hwm_bytes": int(hwm)}, state

    def nothing(ctx):
        return {}

    for cls in args.classes.split(","):
        raw = torch.empty(nraw, dtype=torch.uint8, device="cuda")
        batch.synth_fill(lz4net_b200.default_context(), raw, nraw // synth_bs, synth_bs, synth.CLASS_ID[cls], seed=5)
        out = torch.empty(nraw, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        configs = [(1 << 16, False), (1 << 20, False)] + ([(1 << 20, True)] if cls in ("E50", "ETEXT") else [])
        rows = {}
        for bs, hc in configs:
            row = {}

            def enc_new(ctx, s):
                s["w"] = len(batch.stream_encode_to_host(ctx, raw, bs, hc, dst=wire_new))

            row["encode_new"], s = run(nothing, enc_new)
            w = s["w"]

            def enc_wa(ctx, s):
                hraw.copy_(raw)
                s["w"] = int(l.lz4b200_stream_encode(ctx.handle, hraw.data_ptr(), nraw, bs, int(hc), wire_wa.ctypes.data, cap))

            row["encode_workaround"], s = run(nothing, enc_wa)
            assert s["w"] == w and np.array_equal(wire_new[:w], wire_wa[:w]), (cls, bs, hc)

            def dec_new(ctx, s):
                s["n"] = batch.stream_decode_to_device(ctx, wire_new[:w], out)

            out.zero_()
            row["decode_new"], s = run(nothing, dec_new)
            assert s["n"] == nraw and torch.equal(out, raw), (cls, bs, hc)

            def dec_wa(ctx, s):
                s["n"] = int(l.lz4b200_stream_decode(ctx.handle, wire_wa.ctypes.data, w, hraw.data_ptr(), nraw))
                out.copy_(hraw)
                torch.cuda.synchronize()

            out.zero_()
            row["decode_workaround"], s = run(nothing, dec_wa)
            assert s["n"] == nraw and torch.equal(out, raw), (cls, bs, hc)
            row["wire_bytes"] = w
            row["ratio"] = round(w / nraw, 4)
            key = f"{bs >> 10}KiB-{'hc' if hc else 'fast'}"
            rows[key] = row
            print(cls, key, json.dumps(row), flush=True)
        results["classes"][cls] = rows
        del raw, out
        torch.cuda.empty_cache()
    print(json.dumps(results))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
