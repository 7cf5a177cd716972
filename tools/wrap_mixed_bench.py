"""Times the Wrap / Unwrap calls between device and host memory against the workarounds they replace (host clock around
synchronous work).

    python tools/wrap_mixed_bench.py [--gib 2] [--reps 2] [--classes E0,E50,E100,ETEXT] [--out FILE.json]

For each class, --gib GiB of raw data are generated in HBM and cut into packets of 64 KiB and of 4 KiB (the RPC-sized
case), fast encoder; ETEXT also gets a 64 KiB line with HC.  Every host buffer is page-locked.  Paths, library defaults:
  wrap_new            lz4b200_wrap_batch_packed_from_device: device raw -> packets back to back in host memory
  wrap_dev_compact    lz4b200_wrap_batch_device into worst-case device slots + lz4b200_compact + one D2H copy of the total
  wrap_d2h_host       one D2H copy of the raw bytes + lz4b200_wrap_batch (host -> host slots)
  unwrap_new          lz4b200_unwrap_batch_packed_to_device: host packets -> device raw
  unwrap_h2d_dev      one H2D copy of the packets + lz4b200_unwrap_batch_packed (device)
  unwrap_host_h2d     lz4b200_unwrap_batch (host -> host) + one H2D copy of the raw bytes
Each path runs once on a fresh context (its device-memory high-water mark is read there: free memory before the first
call minus free memory after it, device-wide, with the path's buffers held; the raw data and the unwrap's output tensor
are allocated before and not counted), then --reps times; the mean time per call is reported.  Rates are raw bytes over
time.  Every wrap path's packets are compared with wrap_new's, and every unwrap path's output with the raw data, in the
same run ("equal").  The card's name, power limit, max SM clock and PCIe link are read in the same run.
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


def _slots_equal_packed(slots, stride, plen, packed, off):
    """Packets at i * stride in `slots` (plen[i] bytes each) equal the packets back to back in `packed` (at off[i])."""
    import numpy as np
    n = len(plen)
    rows = slots[:n * stride].reshape(n, stride)
    step = max(1, (256 << 20) // stride)
    for r0 in range(0, n, step):
        r1 = min(n, r0 + step)
        mask = np.arange(stride)[None, :] < plen[r0:r1, None]
        if not np.array_equal(rows[r0:r1][mask], packed[off[r0]:off[r1]]):
            return False
    return True


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
        sys.exit("wrap_mixed_bench.py needs a CUDA device")
    l = native.lib()
    synth_bs = 1 << 20
    nraw = int(args.gib * (1 << 30)) // synth_bs * synth_bs
    card, info = _card()
    results = {"card": card, "power_limit,max_sm_clock,pcie_gen,pcie_width": info, "raw_bytes": nraw,
               "device_hwm": "device-wide, torch.cuda.mem_get_info", "classes": {}}
    most = nraw + 8 * (nraw // 4096)                                    # sum(len + 8) at the smallest packet
    wire_new = torch.empty(most, dtype=torch.uint8).pin_memory().numpy()
    wire_wa = torch.empty(most, dtype=torch.uint8).pin_memory().numpy()
    hraw_t = torch.empty(nraw, dtype=torch.uint8).pin_memory()
    hraw = hraw_t.numpy()

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

    for cls in args.classes.split(","):
        raw = torch.empty(nraw, dtype=torch.uint8, device="cuda")
        batch.synth_fill(lz4net_b200.default_context(), raw, nraw // synth_bs, synth_bs, synth.CLASS_ID[cls], seed=5)
        out = torch.empty(nraw, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        configs = [(1 << 16, False), (1 << 12, False)] + ([(1 << 16, True)] if cls == "ETEXT" else [])
        rows = {}
        for bs, hc in configs:
            n = nraw // bs
            stride = bs + 8
            so = np.arange(n, dtype=np.int64) * bs
            sl = np.full(n, bs, np.int32)
            row = {}

            # ---- wrap: device raw -> packets in host memory ----
            def new_setup(ctx):
                return {"off": np.zeros(n + 1, np.int64), "len": np.zeros(n, np.int32)}

            def wrap_new(ctx, s):
                s["total"] = batch.wrap_to_host_packed(ctx, raw, so, sl, wire_new, s["off"], s["len"], hc=hc)

            row["wrap_new"], s = run(new_setup, wrap_new)
            total, off, plen = s["total"], s["off"], s["len"]
            row["wrap_new"]["equal"] = True

            d_so, d_do, d_sl, d_dc = batch.uniform_layout(n, bs, stride, "cuda")

            def dc_setup(ctx):
                return {"slots": torch.empty(n * stride, dtype=torch.uint8, device="cuda"),
                        "packed": torch.empty(n * stride, dtype=torch.uint8, device="cuda"),
                        "len": torch.zeros(n, dtype=torch.int32, device="cuda"),
                        "off": torch.zeros(n + 1, dtype=torch.int64, device="cuda")}

            def wrap_dc(ctx, s):
                batch.wrap_packed(ctx, raw, d_so, d_sl, s["slots"], d_do, d_dc, s["len"], s["packed"], s["off"], hc=hc)
                k = int(s["off"][n])                                    # (synchronises: the copy needs the total)
                torch.from_numpy(wire_wa[:k]).copy_(s["packed"][:k])
                torch.cuda.synchronize()

            row["wrap_dev_compact"], s = run(dc_setup, wrap_dc)
            row["wrap_dev_compact"]["equal"] = bool(int(s["off"][n]) == total and np.array_equal(wire_wa[:total], wire_new[:total]))
            del s

            h_do = np.arange(n, dtype=np.int64) * stride
            h_dc = np.full(n, stride, np.int32)

            def host_setup(ctx):
                return {"len": np.zeros(n, np.int32)}

            def wrap_host(ctx, s):
                hraw_t.copy_(raw)
                native.check(l.lz4b200_wrap_batch(ctx.handle, hraw.ctypes.data, so.ctypes.data, sl.ctypes.data, int(hc),
                                                  wire_wa.ctypes.data, h_do.ctypes.data, h_dc.ctypes.data,
                                                  s["len"].ctypes.data, n), "wrap_batch")

            row["wrap_d2h_host"], s = run(host_setup, wrap_host)
            row["wrap_d2h_host"]["equal"] = bool(np.array_equal(s["len"], plen)
                                                 and _slots_equal_packed(wire_wa, stride, plen, wire_new, off))

            # ---- unwrap: host packets -> device raw ----
            pstart = off[:-1].copy()

            def un_setup(ctx):
                return {"off": np.zeros(n + 1, np.int64), "res": np.zeros(n, np.int32)}

            def unwrap_new(ctx, s):
                batch.unwrap_to_device_packed(ctx, wire_new, pstart, plen, out, s["off"], s["res"])

            out.zero_()
            row["unwrap_new"], s = run(un_setup, unwrap_new)
            row["unwrap_new"]["equal"] = bool((s["res"] == bs).all() and torch.equal(out, raw))

            def hd_setup(ctx):
                return {"pk": torch.empty(total, dtype=torch.uint8, device="cuda"),
                        "so": torch.from_numpy(pstart).cuda(), "sl": torch.from_numpy(plen).cuda(),
                        "off": torch.zeros(n + 1, dtype=torch.int64, device="cuda"),
                        "res": torch.zeros(n, dtype=torch.int32, device="cuda")}

            wire_t = torch.from_numpy(wire_new[:total])

            def unwrap_hd(ctx, s):
                s["pk"].copy_(wire_t, non_blocking=True)
                batch.unwrap_packed(ctx, s["pk"], s["so"], s["sl"], out, s["off"], s["res"])
                torch.cuda.synchronize()

            out.zero_()
            row["unwrap_h2d_dev"], s = run(hd_setup, unwrap_hd)
            row["unwrap_h2d_dev"]["equal"] = bool(bool((s["res"] == bs).all()) and torch.equal(out, raw))
            del s

            def hh_setup(ctx):
                return {"res": np.zeros(n, np.int32)}

            def unwrap_hh(ctx, s):
                native.check(l.lz4b200_unwrap_batch(ctx.handle, wire_new.ctypes.data, pstart.ctypes.data, plen.ctypes.data,
                                                    hraw.ctypes.data, so.ctypes.data, sl.ctypes.data, s["res"].ctypes.data, n),
                             "unwrap_batch")
                out.copy_(hraw_t, non_blocking=True)
                torch.cuda.synchronize()

            out.zero_()
            row["unwrap_host_h2d"], s = run(hh_setup, unwrap_hh)
            row["unwrap_host_h2d"]["equal"] = bool((s["res"] == bs).all() and torch.equal(out, raw))

            row["packet_bytes"] = total
            row["ratio"] = round(total / nraw, 4)
            key = f"{bs >> 10}KiB-{'hc' if hc else 'fast'}"
            rows[key] = row
            print(cls, key, json.dumps(row), flush=True)
            del d_so, d_do, d_sl, d_dc, wire_t
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
