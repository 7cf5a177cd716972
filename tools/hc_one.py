"""One HC encode of a small E50 batch with each warp kernel (the ncu capture of tools/gpu_hc.sh)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, lz4net_b200
from bench import Workload
ctx = lz4net_b200.Context(0)
nb = torch.cuda.get_device_properties(0).multi_processor_count * 32 * 2
w = Workload(ctx, nb, sys.argv[1] if len(sys.argv) > 1 else "E50", nb, seed=3)
for k in (2, 1):
    ctx.set_option("hc_kernel", k)
    w.encode(hc=True); torch.cuda.synchronize()
print("ok")
