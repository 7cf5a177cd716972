"""Device-timed fast-encode sweep over entropy classes x (CTAs per SM, prefetch distance) -- one GPU process.
usage: python tools/enc_sweep.py [blocks] [classes] [ctas list] [prefetch list] [variant list]
Every configuration is checked: compressed sizes must equal the first configuration's and the round trip must be exact;
the first 64 blocks of every class are also compared byte for byte with the oracle (the checker, never the timed path)."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import lz4net_b200
from bench import Workload, BLOCK, GB

nb = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
CLASSES = sys.argv[2].split(",") if len(sys.argv) > 2 else ("E0", "E50", "E100", "ETEXT")
CTAS = [int(x) for x in sys.argv[3].split(",")] if len(sys.argv) > 3 else (0,)
PF = [int(x) for x in sys.argv[4].split(",")] if len(sys.argv) > 4 else (1024,)
VAR = [int(x) for x in sys.argv[5].split(",")] if len(sys.argv) > 5 else (2,)
ctx = lz4net_b200.Context(0)
peak = 3350.0                       # H100 SXM HBM3, data sheet
for cls in CLASSES:
    w = Workload(ctx, nb, cls, nb, seed=2)
    rb = nb * BLOCK
    ref_len = None
    for ctas, pf, var in [(c, p, v) for v in VAR for c in CTAS for p in PF]:
        if True:
            ctx.set_option("encode_ctas_per_sm", ctas); ctx.set_option("encode_prefetch", pf); ctx.set_option("encode_variant", var)
            w.slots.zero_()
            cs = w.verify()                                            # encode + decode, bit-exact round trip
            lens = w.clen.clone()
            if ref_len is None:
                ref_len = lens
                import numpy as np, oracle
                raw = w.raw[:64 * BLOCK].cpu().numpy(); sl = w.slots[:64 * w.slot].cpu().numpy(); ln = lens[:64].cpu().numpy()
                for b in range(64):
                    r, o = oracle.encode(raw[b * BLOCK:(b + 1) * BLOCK].tobytes())
                    assert r == ln[b] and o == sl[b * w.slot:b * w.slot + r].tobytes(), (cls, b, "not byte-identical to the oracle")
            assert torch.equal(lens, ref_len), (cls, ctas, pf)
            ts = []
            for _ in range(4):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); w.encode(); e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1) * 1e-3)
            t = sorted(ts[1:])[1]
            print(json.dumps({"cls": cls, "ratio": round(cs / rb, 4), "variant": var, "ctas": ctas, "prefetch": pf, "enc_gbs": round(rb / t / GB, 1),
                              "enc_frac": round((rb + cs) / t / GB / peak, 4), "ms": round(t * 1e3, 2)}), flush=True)
    del w; torch.cuda.empty_cache()
