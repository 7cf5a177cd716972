"""Times the host -> host framing calls (lz4b200_stream_encode / stream_decode, lz4b200_wrap_batch / unwrap_batch) of
two builds of the library side by side (host clock around each synchronous call).

    python tools/framing_host_bench.py [--lib NAME=PATH ...] [--gib 2] [--classes E0,E50,E100,ETEXT] [--out FILE.json]

--lib names a build of liblz4b200.so; give it once per build (default: old=build/parent/liblz4b200.so, the library of
an earlier commit built into the git-ignored build/ directory, and new=lz4net_b200/liblz4b200.so).  Each build is loaded
on its own (ctypes, local symbols) and gets a context of its own on device 0.

For each class, --gib GiB of raw data are generated on the device and copied to host memory.  Configurations: LZ4Stream
with 64 KiB and 1 MiB blocks, Wrap with 4 KiB and 64 KiB packets (in slots of packet size + 8); the fast encoder on every
class, HC on E50.  Each configuration runs with every host buffer page-locked and with every host buffer pageable.
Within a configuration each build runs once untimed (its staging buffers grow), then the builds run in turn, twice:
old, new, old, new.  Rates are raw bytes over time.  Every encode's bytes are asserted equal across the builds and every
decode's output equal to the raw data.  "spread" is |run 2 - run 1| / mean of the first build, "ratio" the mean time of
each later build over the first's.  The card's name, power limit, max SM clock and PCIe link are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from mixed_memory_bench import _card  # noqa: E402

_P, _L, _I = C.c_void_p, C.c_int64, C.c_int32


class Build:
    """One liblz4b200.so with a context of its own."""

    def __init__(self, name, path):
        self.name, self.path = name, path
        l = self.l = C.CDLL(path)
        sig = {"lz4b200_create": (C.c_int, [C.POINTER(_P), C.c_int]),
               "lz4b200_destroy": (None, [_P]),
               "lz4b200_last_error": (C.c_char_p, []),
               "lz4b200_stream_bound": (_L, [_L, _I]),
               "lz4b200_stream_encode": (_L, [_P, _P, _L, _I, C.c_int, _P, _L]),
               "lz4b200_stream_decode": (_L, [_P, _P, _L, _P, _L]),
               "lz4b200_wrap_batch": (C.c_int, [_P, _P, _P, _P, C.c_int, _P, _P, _P, _P, _I]),
               "lz4b200_unwrap_batch": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _I]),
               "lz4b200_host_register": (C.c_int, [_P, _L])}
        for fn, (res, args) in sig.items():
            getattr(l, fn).restype, getattr(l, fn).argtypes = res, args
        self.h = _P()
        self.check(l.lz4b200_create(C.byref(self.h), 0), "lz4b200_create")

    def check(self, rc, what):
        if rc < 0:
            raise RuntimeError(f"{self.name}: {what} failed ({rc}): {self.l.lz4b200_last_error().decode()}")
        return rc

    def close(self):
        self.l.lz4b200_destroy(self.h)


def _ptr(a):
    return a.ctypes.data


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--lib", action="append", default=None, metavar="NAME=PATH")
    p.add_argument("--gib", type=float, default=2.0)
    p.add_argument("--classes", default="E0,E50,E100,ETEXT")
    p.add_argument("--out", default=None)
    args = p.parse_args()
    libs = args.lib or [f"old={os.path.join(ROOT, 'build', 'parent', 'liblz4b200.so')}",
                        f"new={os.path.join(ROOT, 'lz4net_b200', 'liblz4b200.so')}"]

    import numpy as np
    import torch
    import lz4net_b200
    from lz4net_b200 import batch, synth
    if not torch.cuda.is_available():
        sys.exit("framing_host_bench.py needs a CUDA device")
    builds = [Build(*s.split("=", 1)) for s in libs]
    synth_bs = 1 << 20
    nraw = int(args.gib * (1 << 30)) // synth_bs * synth_bs
    card, info = _card()
    results = {"card": card, "power_limit,max_sm_clock,pcie_gen,pcie_width": info, "raw_bytes": nraw,
               "builds": {b.name: b.path for b in builds}, "rows": []}
    print(json.dumps({k: results[k] for k in ("card", "power_limit,max_sm_clock,pcie_gen,pcie_width", "builds")}), flush=True)

    big = nraw + nraw // 4096 * 16 + (1 << 20)                     # >= the stream bound and the slots at every size here

    def buffers(pinned):
        def one(n):
            a = np.empty(n, np.uint8)
            if pinned:
                builds[-1].check(builds[-1].l.lz4b200_host_register(_ptr(a), n), "lz4b200_host_register")
            return a
        return {"raw": one(nraw), "dec": one(nraw), "enc": [one(big) for _ in builds]}

    mem = {"pinned": buffers(True), "pageable": buffers(False)}

    def timed(fn):
        t = time.perf_counter()
        fn()
        return (time.perf_counter() - t) * 1e3

    for cls in args.classes.split(","):
        raw_d = torch.empty(nraw, dtype=torch.uint8, device="cuda")
        batch.synth_fill(lz4net_b200.default_context(), raw_d, nraw // synth_bs, synth_bs, synth.CLASS_ID[cls], seed=5)
        torch.cuda.synchronize()
        for m in mem.values():
            torch.from_numpy(m["raw"]).copy_(raw_d)
        del raw_d
        configs = [("stream", 1 << 16, False), ("stream", 1 << 20, False), ("wrap", 1 << 12, False), ("wrap", 1 << 16, False)]
        if cls == "E50":
            configs += [(kind, size, True) for kind, size, _ in configs]
        for kind, size, hc in configs:
            for mname, m in mem.items():
                raw, dec, enc = m["raw"], m["dec"], m["enc"]
                if kind == "stream":
                    wlen = [0] * len(builds)

                    def encode(i):
                        b = builds[i]
                        cap = int(b.l.lz4b200_stream_bound(nraw, size))
                        wlen[i] = b.check(b.l.lz4b200_stream_encode(b.h, _ptr(raw), nraw, size, int(hc), _ptr(enc[i]), cap), "stream_encode")

                    def decode(i):
                        b = builds[i]
                        r = b.check(b.l.lz4b200_stream_decode(b.h, _ptr(enc[i]), wlen[i], _ptr(dec), nraw), "stream_decode")
                        assert r == nraw

                    def same():
                        return all(wlen[i] == wlen[0] and np.array_equal(enc[i][:wlen[0]], enc[0][:wlen[0]])
                                   for i in range(1, len(builds)))

                    wire = lambda: wlen[0]
                else:
                    n = nraw // size
                    stride = size + 8
                    so = np.arange(n, dtype=np.int64) * size
                    sl = np.full(n, size, np.int32)
                    po = np.arange(n, dtype=np.int64) * stride
                    pc = np.full(n, stride, np.int32)
                    plen = [np.zeros(n, np.int32) for _ in builds]
                    res = np.zeros(n, np.int32)

                    def encode(i):
                        b = builds[i]
                        b.check(b.l.lz4b200_wrap_batch(b.h, _ptr(raw), _ptr(so), _ptr(sl), int(hc), _ptr(enc[i]), _ptr(po),
                                                       _ptr(pc), _ptr(plen[i]), n), "wrap_batch")

                    def decode(i):
                        b = builds[i]
                        res[:] = 0
                        b.check(b.l.lz4b200_unwrap_batch(b.h, _ptr(enc[i]), _ptr(po), _ptr(plen[i]), _ptr(dec), _ptr(so),
                                                         _ptr(sl), _ptr(res), n), "unwrap_batch")
                        assert (res == size).all()

                    def same():
                        # the packets, not the bytes behind them in their slots
                        if not all(np.array_equal(plen[i], plen[0]) for i in range(1, len(builds))):
                            return False
                        rows = [e[:n * stride].reshape(n, stride) for e in enc]
                        step = max(1, (256 << 20) // stride)
                        for r0 in range(0, n, step):
                            mask = np.arange(stride)[None, :] < plen[0][r0:r0 + step, None]
                            if not all(np.array_equal(r[r0:r0 + step][mask], rows[0][r0:r0 + step][mask]) for r in rows[1:]):
                                return False
                        return True

                    wire = lambda: int(plen[0].sum())
                row = {"class": cls, "call": kind, "size_kib": size >> 10, "mode": "hc" if hc else "fast", "memory": mname}
                for op, fn in (("encode", encode), ("decode", decode)):
                    ms = {b.name: [] for b in builds}
                    for i in range(len(builds)):
                        fn(i)                                               # untimed: staging buffers grow
                        if op == "decode":
                            assert np.array_equal(dec, raw), (builds[i].name, cls, kind, size, hc, mname)
                    for _ in range(2):
                        for i, b in enumerate(builds):
                            if op == "decode":
                                dec[:1] = ~raw[:1]                          # (a decode that writes nothing fails)
                            ms[b.name].append(timed(lambda: fn(i)))
                            if op == "decode":
                                assert np.array_equal(dec, raw), (b.name, cls, kind, size, hc, mname)
                    if op == "encode":
                        assert same(), (cls, kind, size, hc, mname)
                    first = ms[builds[0].name]
                    mean0 = sum(first) / 2
                    row[op] = {"ms": {k: [round(x, 1) for x in v] for k, v in ms.items()},
                               "raw_gbs": {k: round(nraw / (sum(v) / 2) / 1e6, 2) for k, v in ms.items()},
                               "spread": round(abs(first[1] - first[0]) / mean0, 3),
                               "ratio": {k: round(sum(v) / 2 / mean0, 3) for k, v in ms.items() if k != builds[0].name}}
                row["ratio_wire"] = round(wire() / nraw, 4)
                results["rows"].append(row)
                print(json.dumps(row), flush=True)
    for b in builds:
        b.close()
    print(json.dumps(results))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
