"""Times the mixed-memory batch calls against the workarounds they replace (host clock around synchronous work).

    python tools/mixed_memory_bench.py [--blocks 32768] [--reps 3] [--classes E0,E50,E100,ETEXT] [--out FILE.json]

For each class, --blocks x 64 KiB blocks are generated on the device; the compressed side on the host is page-locked.
Paths, fast encoder, library defaults:
  d2h_encode          lz4b200_encode_batch_packed_from_device: device raw -> packed compressed bytes in host memory
  d2h_workaround      lz4b200_encode_batch(MEM_DEVICE) into worst-case slots + lz4b200_compact + one D2H copy of the total
  h2d_decode          lz4b200_decode_batch(MEM_HOST_TO_DEVICE), known size: host compressed -> device raw
  h2d_copy_decode     one H2D copy of the packed compressed bytes + lz4b200_decode_batch(MEM_DEVICE)
  h2d_host_decode     lz4b200_decode_batch(MEM_HOST) into host raw + one H2D copy of the raw bytes
Each path runs once on a fresh context (its device-memory high-water mark is read there), then --reps times; the mean
time per call is reported.  Rates are raw bytes over time.  pcie_bytes counts the payload each path moves over the host
link, from the sizes (the per-block metadata is left out).  device_hwm_bytes is device-wide (torch.cuda.mem_get_info):
free memory before the first call minus free memory after it, with torch's cache emptied before and the path's tensors
still held after; the source data is allocated before and not counted.  Every path's output is checked against the
others'.  The card's name, power limit, max SM clock and PCIe link are read in the same run.
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
        q = "power.limit,clocks.max.sm,pcie.link.gen.current,pcie.link.width.current"
        info = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        info = "unknown"
    return name, info


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--blocks", type=int, default=1 << 15)
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--classes", default="E0,E50,E100,ETEXT")
    p.add_argument("--out", default=None)
    args = p.parse_args()

    import numpy as np
    import torch
    import lz4net_b200
    from lz4net_b200 import batch, synth
    if not torch.cuda.is_available():
        sys.exit("mixed_memory_bench.py needs a CUDA device")
    nb, bs = args.blocks, 65536
    slot = bs + bs // 255 + 16
    card, info = _card()
    results = {"card": card, "power_limit,max_sm_clock,pcie_gen,pcie_width": info, "blocks": nb, "block_size": bs,
               "device_hwm": "device-wide, torch.cuda.mem_get_info", "classes": {}}
    so = np.arange(nb, dtype=np.int64) * bs
    sl = np.full(nb, bs, np.int32)
    caps = np.full(nb, slot, np.int32)
    d_so, d_do, d_sl, d_dc = batch.uniform_layout(nb, bs, slot, "cuda")

    def run(setup, fn, raw_bytes):
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
        return {"ms": round(ms, 2), "raw_gbs": round(raw_bytes / ms / 1e6, 2), "device_hwm_bytes": int(hwm)}, state

    for cls in args.classes.split(","):
        raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
        batch.synth_fill(lz4net_b200.default_context(), raw, nb, bs, synth.CLASS_ID[cls], seed=5)
        torch.cuda.synchronize()
        nraw = nb * bs
        hcomp = torch.empty(nb * slot, dtype=torch.uint8).pin_memory().numpy()
        row = {}

        # ---- device -> host encode ----
        def d2h_setup(ctx):
            return {"off": np.zeros(nb + 1, np.int64), "len": np.zeros(nb, np.int32)}

        def d2h(ctx, s):
            s["total"] = batch.encode_to_host_packed(ctx, raw, so, sl, caps, hcomp, s["off"], s["len"])

        r, s_new = run(d2h_setup, d2h, nraw)
        total = s_new["total"]
        coff, clen = s_new["off"], s_new["len"]
        r["pcie_bytes"] = total
        row["d2h_encode"] = r

        hwork = torch.empty(nb * slot, dtype=torch.uint8).pin_memory()

        def wa_setup(ctx):
            return {"slots": torch.empty(nb * slot, dtype=torch.uint8, device="cuda"),
                    "packed": torch.empty(nb * slot, dtype=torch.uint8, device="cuda"),
                    "len": torch.zeros(nb, dtype=torch.int32, device="cuda"),
                    "off": torch.zeros(nb + 1, dtype=torch.int64, device="cuda")}

        def wa(ctx, s):
            batch.encode(ctx, raw, d_so, d_sl, s["slots"], d_do, d_dc, s["len"])
            batch.compact(ctx, s["slots"], d_do, s["len"], s["packed"], s["off"])
            n = int(s["off"][nb])                                    # (synchronises: the copy needs the total)
            hwork[:n].copy_(s["packed"][:n])
            torch.cuda.synchronize()

        r, s_wa = run(wa_setup, wa, nraw)
        r["pcie_bytes"] = total
        row["d2h_workaround"] = r
        assert np.array_equal(s_wa["len"].cpu().numpy(), clen) and np.array_equal(hwork[:total].numpy(), hcomp[:total]), cls
        del s_wa, hwork

        # ---- host -> device decode (known size) ----
        dst_off = so
        cstart = coff[:-1].copy()

        def h2d_setup(ctx):
            return {"out": torch.empty(nraw, dtype=torch.uint8, device="cuda"), "res": np.zeros(nb, np.int32)}

        def h2d(ctx, s):
            batch.decode_from_host(ctx, hcomp, cstart, clen, s["out"], dst_off, sl, s["res"])

        r, s = run(h2d_setup, h2d, nraw)
        assert np.array_equal(s["res"], clen) and torch.equal(s["out"], raw), cls
        r["pcie_bytes"] = total
        row["h2d_decode"] = r
        del s

        def cd_setup(ctx):
            return {"comp": torch.empty(total, dtype=torch.uint8, device="cuda"),
                    "out": torch.empty(nraw, dtype=torch.uint8, device="cuda"),
                    "res": torch.zeros(nb, dtype=torch.int32, device="cuda"),
                    "off": torch.from_numpy(cstart).cuda(), "len": torch.from_numpy(clen).cuda()}

        hcomp_t = torch.from_numpy(hcomp[:total])

        def cd(ctx, s):
            s["comp"].copy_(hcomp_t, non_blocking=True)
            batch.decode(ctx, s["comp"], s["off"], s["len"], s["out"], d_so, d_sl, s["res"])
            torch.cuda.synchronize()

        r, s = run(cd_setup, cd, nraw)
        assert torch.equal(s["res"].cpu(), torch.from_numpy(clen)) and torch.equal(s["out"], raw), cls
        r["pcie_bytes"] = total
        row["h2d_copy_decode"] = r
        del s

        hraw = torch.empty(nraw, dtype=torch.uint8).pin_memory()

        def hd_setup(ctx):
            return {"out": torch.empty(nraw, dtype=torch.uint8, device="cuda"), "res": np.zeros(nb, np.int32)}

        def hd(ctx, s):
            ctx.decode_batch_ptr(hcomp.ctypes.data, cstart.ctypes.data, clen.ctypes.data, hraw.data_ptr(), so.ctypes.data,
                                 sl.ctypes.data, s["res"].ctypes.data, nb, known=True, device=False)
            s["out"].copy_(hraw, non_blocking=True)
            torch.cuda.synchronize()

        r, s = run(hd_setup, hd, nraw)
        assert np.array_equal(s["res"], clen) and torch.equal(s["out"], raw), cls
        r["pcie_bytes"] = total + 2 * nraw                           # compressed up, raw down, raw up again
        row["h2d_host_decode"] = r
        del s, hraw

        row["ratio"] = round(total / nraw, 4)
        results["classes"][cls] = row
        print(cls, json.dumps(row), flush=True)
        del raw, hcomp, hcomp_t
        torch.cuda.empty_cache()
    print(json.dumps(results))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
