"""Times the packed unknown-size decode from host memory into device memory against what a caller could do without it
(host clock around synchronous work).

    python tools/packed_mixed_bench.py [--mib 2048] [--reps 3] [--rows E0:65536:pinned,...] [--out FILE.json]

A row is class:block_size:pinned|pageable.  Default rows: E0, E50, E100 and ETEXT as 64 KiB blocks from page-locked memory,
E50 as 4 KiB blocks, and E50 as 64 KiB blocks from pageable memory.  For each row --mib MiB of raw data are generated and
fast-encoded on the device into packed compressed bytes in host memory; only the compressed lengths are kept.  Paths:
  packed_to_device    lz4b200_decode_batch_packed_to_device: one call, the compressed bytes cross PCIe once
  measure_then_decode lz4b200_measure_batch(MEM_HOST) + a prefix sum on the host + lz4b200_decode_batch(MEM_HOST_TO_DEVICE,
                      known_len = 0): the compressed bytes cross PCIe twice
  copy_then_packed    one H2D copy of the whole compressed batch (and its offsets and lengths) + lz4b200_decode_batch_packed:
                      the compressed batch is held in device memory
  known_size          lz4b200_decode_batch(MEM_HOST_TO_DEVICE, known_len = 1) with the decoded sizes given: what storing
                      the sizes would buy
Each path runs once, untimed, on a fresh context of its own (its device-memory high-water mark is read there: device-wide
free memory before the context minus after the call, torch's cache emptied before, the path's tensors -- its output, and
copy_then_packed's device copy of the batch -- held); then the paths are run in turn, --reps rounds, and every call's time
is reported.  Rates are raw bytes over time.  pcie_bytes is the payload a path moves over the host link, from the sizes
(per-block metadata left out).  Every path's output is compared with the source data, so all paths produce identical
bytes.  The card's name, power limit, max SM clock and PCIe link are read in the same run.
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

DEFAULT_ROWS = "E0:65536:pinned,E50:65536:pinned,E100:65536:pinned,ETEXT:65536:pinned,E50:4096:pinned,E50:65536:pageable"


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
    p.add_argument("--mib", type=int, default=2048)
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--rows", default=DEFAULT_ROWS)
    p.add_argument("--out", default=None)
    args = p.parse_args()
    rows = []
    for r in args.rows.split(","):
        cls, bs, mem = r.split(":")
        if mem not in ("pinned", "pageable") or int(bs) < 1:
            sys.exit(f"bad row {r!r}: class:block_size:pinned|pageable")
        rows.append((cls, int(bs), mem == "pinned"))

    import numpy as np
    import torch
    import lz4net_b200
    from lz4net_b200 import batch, synth
    if not torch.cuda.is_available():
        sys.exit("packed_mixed_bench.py needs a CUDA device")
    card, info = _card()
    results = {"card": card, "power_limit,max_sm_clock,pcie_gen,pcie_width": info, "raw_mib": args.mib, "reps": args.reps,
               "device_hwm": "device-wide, torch.cuda.mem_get_info", "rows": []}
    print(json.dumps({k: results[k] for k in ("card", "power_limit,max_sm_clock,pcie_gen,pcie_width")}), flush=True)

    for cls, bs, pinned in rows:
        nb = (args.mib << 20) // bs
        nraw = nb * bs
        slot = bs + bs // 255 + 16
        raw = torch.empty(nraw, dtype=torch.uint8, device="cuda")
        batch.synth_fill(lz4net_b200.default_context(), raw, nb, bs, synth.CLASS_ID[cls], seed=5)
        so = np.arange(nb, dtype=np.int64) * bs
        sl = np.full(nb, bs, np.int32)
        hcomp = torch.empty(nb * slot, dtype=torch.uint8).pin_memory().numpy()
        coff, clen = np.zeros(nb + 1, np.int64), np.zeros(nb, np.int32)
        total = batch.encode_to_host_packed(lz4net_b200.default_context(), raw, so, sl, np.full(nb, slot, np.int32), hcomp, coff, clen)
        cstart = coff[:-1].copy()
        if not pinned:
            hcomp = hcomp[:total + 16].copy()                         # a plain numpy array: pageable
        hcomp_t = torch.from_numpy(hcomp[:total])

        def new_out():
            return {"out": torch.zeros(nraw, dtype=torch.uint8, device="cuda"), "off": np.zeros(nb + 1, np.int64),
                    "res": np.zeros(nb, np.int32)}

        def packed_to_device(ctx, s):
            batch.decode_from_host_packed(ctx, hcomp, cstart, clen, s["out"], s["off"], s["res"])

        def measure_then_decode(ctx, s):
            ctx.measure_batch_ptr(hcomp.ctypes.data, cstart.ctypes.data, clen.ctypes.data, None, s["res"].ctypes.data, nb,
                                  known=False, device=False)
            caps = np.maximum(s["res"], 0)
            s["off"][0] = 0
            np.cumsum(caps, dtype=np.int64, out=s["off"][1:])
            batch.decode_from_host(ctx, hcomp, cstart, clen, s["out"], s["off"][:-1], caps, s["res"], known=False)

        def copy_setup():
            s = new_out()
            s.update(comp=torch.empty(total, dtype=torch.uint8, device="cuda"), d_so=torch.empty(nb, dtype=torch.int64, device="cuda"),
                     d_sl=torch.empty(nb, dtype=torch.int32, device="cuda"), d_off=torch.zeros(nb + 1, dtype=torch.int64, device="cuda"),
                     d_res=torch.zeros(nb, dtype=torch.int32, device="cuda"))
            return s

        def copy_then_packed(ctx, s):
            s["comp"].copy_(hcomp_t, non_blocking=True)
            s["d_so"].copy_(torch.from_numpy(cstart), non_blocking=True)
            s["d_sl"].copy_(torch.from_numpy(clen), non_blocking=True)
            batch.decode_packed(ctx, s["comp"], s["d_so"], s["d_sl"], s["out"], s["d_off"], s["d_res"])
            s["off"][:] = s["d_off"].cpu().numpy()                    # (synchronises: the caller wants offsets and results)
            s["res"][:] = s["d_res"].cpu().numpy()

        def known_size(ctx, s):
            batch.decode_from_host(ctx, hcomp, cstart, clen, s["out"], so, sl, s["res"], known=True)
            s["off"][:-1] = so
            s["off"][-1] = nraw

        paths = [("packed_to_device", new_out, packed_to_device, total), ("measure_then_decode", new_out, measure_then_decode, 2 * total),
                 ("copy_then_packed", copy_setup, copy_then_packed, total), ("known_size", new_out, known_size, total)]
        live = []
        row = {"class": cls, "block_size": bs, "blocks": nb, "source": "page-locked" if pinned else "pageable",
               "ratio": round(total / nraw, 4), "paths": {}}
        for name, setup, fn, pcie in paths:
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            free0 = torch.cuda.mem_get_info()[0]
            ctx = lz4net_b200.Context(0)
            s = setup()
            fn(ctx, s)
            torch.cuda.synchronize()
            hwm = free0 - torch.cuda.mem_get_info()[0]
            want_res = clen if name == "known_size" else sl
            assert np.array_equal(s["res"], want_res) and np.array_equal(s["off"], np.arange(nb + 1, dtype=np.int64) * bs), (cls, name)
            assert torch.equal(s["out"], raw), (cls, name)
            row["paths"][name] = {"pcie_bytes": int(pcie), "device_hwm_bytes": int(hwm), "ms": []}
            live.append((name, ctx, s, fn))
        for _ in range(args.reps):
            for name, ctx, s, fn in live:
                s["out"].zero_()
                torch.cuda.synchronize()
                t = time.perf_counter()
                fn(ctx, s)
                torch.cuda.synchronize()
                row["paths"][name]["ms"].append(round((time.perf_counter() - t) * 1e3, 2))
                assert torch.equal(s["out"], raw), (cls, name)
        for name, ctx, s, fn in live:
            r = row["paths"][name]
            r["raw_gbs"] = [round(nraw / ms / 1e6, 2) for ms in r["ms"]]
            ctx.close()
        results["rows"].append(row)
        print(json.dumps(row), flush=True)
        del live, raw, hcomp, hcomp_t, s
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
