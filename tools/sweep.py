"""Device-timed decode/encode sweep over entropy classes and tuning knobs (one GPU process).
usage: python tools/sweep.py [blocks]"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import lz4net_b200
from bench import Workload, measure_pair, BLOCK, GB

nb = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
ctx = lz4net_b200.Context(0)
peak = 3350.0                       # H100 SXM HBM3, data sheet
res = {}
CLASSES = sys.argv[2].split(",") if len(sys.argv) > 2 else ("E0", "E50", "E100", "ETEXT")
ENC = len(sys.argv) <= 3 or sys.argv[3] == "enc"
for cls in CLASSES:
    w = Workload(ctx, nb, cls, nb, seed=2)
    cs = w.verify(); rb = nb * BLOCK
    row = {"ratio": round(cs / rb, 4)}
    LANES = [int(x) for x in sys.argv[4].split(",")] if len(sys.argv) > 4 else (32, 16, 8, 132, 116, 108)
    for lanes in LANES:
        ctx.set_option("decode_lanes", lanes)
        # correctness under this lane count
        for wv in range(w.n_waves):
            b0, b1 = w.decode_wave(wv); torch.cuda.synchronize()
            assert torch.equal(w.out[:(b1 - b0) * BLOCK], w.raw[b0 * BLOCK:b1 * BLOCK]), (cls, lanes)
        torch.cuda.synchronize()
        ts = []
        for _ in range(5):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for wv in range(w.n_waves):
                w.decode_wave(wv)
            e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1) * 1e-3)
        t = sorted(ts)[len(ts) // 2]
        row[f"dec{lanes}_gbs"] = round(rb / t / GB, 1); row[f"dec{lanes}_frac"] = round((rb + cs) / t / GB / peak, 3)
    ctx.set_option("decode_lanes", 32)
    for ctas in ((0,) if ENC else ()):
        ctx.set_option("encode_ctas_per_sm", ctas)
        ts = []
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); w.encode(); e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1) * 1e-3)
        row[f"enc_ctas{ctas}_gbs"] = round(rb / sorted(ts)[1] / GB, 1)
    ctx.set_option("encode_ctas_per_sm", 0)
    res[cls] = row
    print(cls, json.dumps(row), flush=True)
    del w; torch.cuda.empty_cache()
