"""LZ4HC on blocks above 64 KiB: the default (blocks above 64 KiB on the window kernel, lz4hc_window.cuh) against hc_kernel 0
(a thread per block), alternating default / 0 / default in one process.  Device-timed batches of 128 KiB, 1 MiB and 4 MiB
blocks of E50 / ETEXT / TEXT (blocks cut from this repository's own documents, tiled); the mixed 1-in-4 x 128 KiB batch;
the latency of one 1 MiB EncodeHC; a 1 GiB stream_encode with HighCompression at 1 MiB blocks from host memory; the same
blocks on the host cores (oracle/_ref when built, else the port).  Every configuration's lengths are compared with the
default's.  Prints one line per measurement; --out also writes them all to a JSON file.

usage: hc_window_ab.py [--budget SECONDS] [--out FILE.json] [--rows CLASS:BLOCKS:BLOCK_BYTES,...] [--no-latency] [--no-stream]
       (CLASS: E50, ETEXT, TEXT or MIXED_E50 = one block in four at full size, the others cut to 64 KiB)"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import lz4net_b200
import oracle
from lz4net_b200 import batch, synth

ap = argparse.ArgumentParser()
ap.add_argument("--budget", type=float, default=900.0, help="seconds after which no new measurement is started")
ap.add_argument("--out", default=None)
ap.add_argument("--rows", default=None)
ap.add_argument("--no-latency", action="store_true")
ap.add_argument("--no-stream", action="store_true")
ap.add_argument("--stream-kernels", default="-1,0,-1", help="hc_kernel values the 1 GiB stream_encode is timed with, in turn")
args = ap.parse_args()
T0 = time.time()
budget = args.budget
GB = 1e9
ctx = lz4net_b200.Context(0)
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"device": torch.cuda.get_device_name(0), "nvidia_smi": smi, "runs": []}


def save():
    if args.out:
        json.dump(out, open(args.out, "w"), indent=1)


def text_bytes(n):
    data = b""
    for name in ("SURVEY.md", "DESIGN.md", "BASELINE.md", "INTEGRATION.md", "README.md", "bench.py", "lz4net_b200/csrc/capi.cu"):
        data += open(os.path.join(ROOT, name), "rb").read()
    return np.frombuffer((data * (n // len(data) + 1))[:n], np.uint8)


def make(cls, nb, bs, lens=None):
    raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    if cls == "TEXT":
        t = torch.from_numpy(text_bytes(min(nb, 64) * bs).copy()).cuda().view(-1, bs)
        raw.view(nb, bs).copy_(t.repeat((nb + t.shape[0] - 1) // t.shape[0], 1)[:nb])
    else:
        batch.synth_fill(ctx, raw, nb * (bs // 65536), 65536, synth.CLASS_ID[cls], seed=3, first_block=0)
    slot = oracle.bound(bs)
    so, do, sl, dc = batch.uniform_layout(nb, bs, slot, "cuda")
    if lens is not None:
        sl = sl.clone(); sl[torch.arange(nb, device="cuda") % 4 != 0] = lens
    slots = torch.empty(nb * slot, dtype=torch.uint8, device="cuda")
    clen = torch.zeros(nb, dtype=torch.int32, device="cuda")
    return raw, so, sl, slots, do, dc, clen


def timed(w, kernel):
    ctx.set_option("hc_kernel", kernel)
    raw, so, sl, slots, do, dc, clen = w
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); batch.encode(ctx, raw, so, sl, slots, do, dc, clen, hc=True); e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3, clen.clone()


WORK = [("E50", 256, 1 << 17), ("ETEXT", 256, 1 << 17), ("TEXT", 256, 1 << 17),
        ("E50", 256, 1 << 20), ("ETEXT", 256, 1 << 20), ("TEXT", 256, 1 << 20),
        ("E50", 256, 4 << 20), ("ETEXT", 256, 4 << 20), ("TEXT", 256, 4 << 20),
        ("E50", 4096, 1 << 17), ("ETEXT", 4096, 1 << 17), ("TEXT", 4096, 1 << 17),
        ("E50", 4096, 1 << 20), ("ETEXT", 4096, 1 << 20), ("TEXT", 4096, 1 << 20),
        ("MIXED_E50", 4096, 1 << 17)]
if args.rows:
    WORK = [(c, int(nb), int(bs)) for c, nb, bs in (r.split(":") for r in args.rows.split(","))]
for cls, nb, bs in WORK:
    if time.time() - T0 > budget:
        out["skipped_from"] = [cls, nb, bs]; break
    w = make(cls.replace("MIXED_", ""), nb, bs, 65536 if cls.startswith("MIXED") else None)
    raw_bytes = int(w[2].sum())
    timed(w, -1)                                                        # warm-up (arena, modules)
    t_a, len_a = timed(w, -1)
    t_0, len_0 = timed(w, 0)
    t_b, len_b = timed(w, -1)
    row = {"class": cls, "blocks": nb, "block": bs, "default_s": round(min(t_a, t_b), 4), "thread_s": round(t_0, 4),
           "default_gbs": round(raw_bytes / min(t_a, t_b) / GB, 3), "thread_gbs": round(raw_bytes / t_0 / GB, 3),
           "same_lengths": bool(torch.equal(len_a, len_0) and torch.equal(len_a, len_b)),
           "ratio": round(int(len_a.sum()) / raw_bytes, 4)}
    if nb == 256 and time.time() - T0 < budget:                         # the same blocks on the host cores
        k = 16 if bs <= (1 << 20) else 8
        h = w[0][: k * bs].cpu().numpy()
        slot = oracle.bound(bs)
        so = np.arange(k, dtype=np.int64) * bs; do = np.arange(k, dtype=np.int64) * slot
        sl = np.full(k, bs, np.int32); dc = np.full(k, slot, np.int32)
        comp = np.zeros(k * slot + 64, np.uint8)
        impl = "ref" if oracle.have_ref() else "port"
        t, _ = oracle.mt_run("encode_hc", impl, h, so, sl, comp, do, dc, os.cpu_count() or 1)
        row["cpu_gbs"] = round(k * bs / t / GB, 3); row["cpu_impl"] = impl; row["cpu_threads"] = os.cpu_count()
    out["runs"].append(row); print(row, flush=True); save()
    del w; torch.cuda.empty_cache()

ctx.set_option("hc_kernel", -1)
if not args.no_latency and time.time() - T0 < budget:
    # one 1 MiB block from host memory per call, host-timed: the path of the single-block EncodeHC (whose own per-thread
    # context does not take options, hence a one-block batch on this one)
    d = text_bytes(1 << 20).tobytes()
    lat = {}
    for k in (-1, 0, -1):
        ctx.set_option("hc_kernel", k)
        if k == -1:
            ctx.encode_blocks([d], hc=True)                            # warm-up (the thread kernel's takes as long as its timed call)
        t0 = time.time(); r, _ = ctx.encode_blocks([d], hc=True); lat.setdefault(str(k), []).append(round(time.time() - t0, 4))
        assert r[0] == oracle.encode_hc(d)[0]
    ctx.set_option("hc_kernel", -1)
    out["encodehc_1mib_text_latency_s"] = lat; print(lat, flush=True); save()

if not args.no_stream and time.time() - T0 < budget:
    data = bytearray()
    for i in range(1024):                                              # 1 GiB: E50 / ETEXT / text chunks in turn
        data += synth.make_blocks(("E50", "ETEXT")[i % 2], 16, 65536, seed=i).tobytes() if i % 3 else text_bytes(1 << 20).tobytes()
    data = bytes(data)
    res = {}
    for k in (int(v) for v in args.stream_kernels.split(",")):
        if k == 0 and time.time() - T0 > budget:
            continue
        ctx.set_option("hc_kernel", k)
        t0 = time.time(); s = ctx.stream_encode(data, 1 << 20, high_compression=True); dt = time.time() - t0
        res.setdefault(str(k), []).append({"s": round(dt, 3), "gbs": round(len(data) / dt / GB, 3), "bytes": len(s)})
    ctx.set_option("hc_kernel", -1)
    out["stream_encode_1gib_hc_1mib"] = res; print(res, flush=True)
out["seconds"] = round(time.time() - T0, 1)
save()
print("done in", out["seconds"], "s", flush=True)
