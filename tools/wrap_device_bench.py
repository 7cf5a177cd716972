"""Times the Wrap / Unwrap packets in device memory against the codec calls they wrap (CUDA events).

    python tools/wrap_device_bench.py [--blocks 131072] [--reps 5] [--classes E0,E50,E100,ETEXT] [--host-blocks 16384] [--out FILE.json]

For each class, 2^17 x 64 KiB blocks are generated on the device; then each call below runs `--reps` times after a warm-up
and the mean time per call is reported:
  encode         lz4b200_encode_batch(MEM_DEVICE), fast, capacity = block length (what Wrap gives the encoder)
  wrap           lz4b200_wrap_batch_device, fast, into slots of block + 8 bytes
  known          lz4b200_decode_batch(MEM_DEVICE), known size, of the packets' compressed payloads
  unwrap         lz4b200_unwrap_batch_device of the packets
  unwrap_packed  lz4b200_unwrap_batch_packed of the packets
  host_wrap / host_unwrap  lz4b200_wrap_batch / unwrap_batch from and to pinned host memory, over the first --host-blocks
                 blocks (host clock around the synchronous call)
Rates are raw bytes over time.  wrap_over_encode and unwrap_over_known are the framing's overhead.  Every call's results
are checked (the packets equal the encode + stored-raw rule; the unwrapped bytes equal the input).  The card's name and
power limit are printed with the numbers.
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


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--blocks", type=int, default=1 << 17)
    p.add_argument("--reps", type=int, default=5)
    p.add_argument("--classes", default="E0,E50,E100,ETEXT")
    p.add_argument("--host-blocks", type=int, default=1 << 14)
    p.add_argument("--out", default=None)
    args = p.parse_args()

    import numpy as np
    import torch
    import lz4net_b200
    from lz4net_b200 import batch, native, synth
    if not torch.cuda.is_available():
        sys.exit("wrap_device_bench.py needs a CUDA device")
    ctx = lz4net_b200.default_context()
    nb, bs = args.blocks, 65536
    card, power = _card()
    results = {"card": card, "power_limit_and_max_sm_clock": power, "blocks": nb, "block_size": bs, "classes": {}}

    def timed(fn):
        fn()                                                        # warm-up
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.reps):
            fn()
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1) / args.reps

    def host_timed(fn):
        fn()
        t = time.perf_counter()
        for _ in range(args.reps):
            fn()
        return (time.perf_counter() - t) * 1e3 / args.reps

    for cls in args.classes.split(","):
        raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
        batch.synth_fill(ctx, raw, nb, bs, synth.CLASS_ID[cls], seed=5)
        so, do, sl, _ = batch.uniform_layout(nb, bs, bs + 8, "cuda")
        pay = do + 8
        slots = torch.empty(nb * (bs + 8), dtype=torch.uint8, device="cuda")
        caps = sl + 8
        clen = torch.zeros(nb, dtype=torch.int32, device="cuda")
        plen = torch.zeros(nb, dtype=torch.int32, device="cuda")
        t = {
            "encode": timed(lambda: batch.encode(ctx, raw, so, sl, slots, pay, sl, clen)),
            "wrap": timed(lambda: batch.wrap(ctx, raw, so, sl, slots, do, caps, plen)),
        }
        torch.cuda.synchronize()
        stored = torch.where((clen <= 0) | (clen >= bs), torch.full_like(clen, bs), clen)
        assert torch.equal(plen, stored + 8), cls
        comp = stored < bs                                          # the packets the decoder sees
        out = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
        res = torch.zeros(nb, dtype=torch.int32, device="cuda")
        out_off = torch.zeros(nb + 1, dtype=torch.int64, device="cuda")
        dl = torch.where(comp, stored, torch.zeros_like(stored))
        dc = torch.where(comp, sl, torch.zeros_like(sl))
        t["known"] = timed(lambda: batch.decode(ctx, slots, pay, dl, out, so, dc, res, known=True))
        t["unwrap"] = timed(lambda: batch.unwrap(ctx, slots, do, plen, out, so, sl, res))
        torch.cuda.synchronize()
        assert bool((res == bs).all()) and torch.equal(out, raw), cls
        out.zero_()
        t["unwrap_packed"] = timed(lambda: batch.unwrap_packed(ctx, slots, do, plen, out, out_off, res))
        torch.cuda.synchronize()
        assert bool((res == bs).all()) and torch.equal(out, raw), cls
        # host framing from pinned memory, for context
        hb = min(args.host_blocks, nb)
        hraw = raw[:hb * bs].cpu().pin_memory()
        hpk = torch.empty(hb * (bs + 8), dtype=torch.uint8).pin_memory()
        hout = torch.empty(hb * bs, dtype=torch.uint8).pin_memory()
        hso = np.arange(hb, dtype=np.int64) * bs
        hdo = np.arange(hb, dtype=np.int64) * (bs + 8)
        hsl = np.full(hb, bs, np.int32); hcap = hsl + 8
        hpl = np.zeros(hb, np.int32); hres = np.zeros(hb, np.int32)
        l = native.lib()
        t["host_wrap"] = host_timed(lambda: native.check(l.lz4b200_wrap_batch(
            ctx.handle, hraw.data_ptr(), hso.ctypes.data, hsl.ctypes.data, 0, hpk.data_ptr(), hdo.ctypes.data, hcap.ctypes.data,
            hpl.ctypes.data, hb), "wrap_batch"))
        t["host_unwrap"] = host_timed(lambda: native.check(l.lz4b200_unwrap_batch(
            ctx.handle, hpk.data_ptr(), hdo.ctypes.data, hpl.ctypes.data, hout.data_ptr(), hso.ctypes.data, hsl.ctypes.data,
            hres.ctypes.data, hb), "unwrap_batch"))
        assert (hres == bs).all() and torch.equal(hout, hraw), cls
        ratio = float(plen.sum()) / (nb * (bs + 8))
        row = {"packet_ratio": round(ratio, 4), "stored_packets": int((~comp).sum())}
        for k, ms in t.items():
            n_bytes = (hb if k.startswith("host") else nb) * bs
            row[k + "_ms"] = round(ms, 3)
            row[k + "_gbs"] = round(n_bytes / ms / 1e6, 1)
        row["wrap_over_encode"] = round(t["wrap"] / t["encode"], 3)
        row["unwrap_over_known"] = round(t["unwrap"] / t["known"], 3)
        row["unwrap_packed_over_known"] = round(t["unwrap_packed"] / t["known"], 3)
        results["classes"][cls] = row
        print(cls, json.dumps(row), flush=True)
        del raw, slots, out, hraw, hpk, hout
        torch.cuda.empty_cache()
    print(json.dumps(results))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
