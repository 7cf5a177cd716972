"""Where the fast encoder's time goes, per sequence: event counts and clock64 cycles per phase (lz4net_b200/csrc/enc_prof.cuh).

    python tools/enc_phases.py [--blocks N] [--cls E50,ETEXT] [--reps R] [--out FILE.json]   # H100: instrumented kernel
    python tools/enc_phases.py --emu [--blocks N] [--cls E50,ETEXT]                         # CPU emulator: events only

The GPU mode builds the kernel twice into a temporary directory, with the counters and without, times both on the same
batch (CUDA events) and prints per sequence: rounds, exact-path rounds, probe hits, ... and the cycles of each phase,
summed over the warps.  The uninstrumented time shows what the counters themselves cost.  Blocks are 64 KiB of the
synthetic classes of lz4net_b200/synth.py, seed 2.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lz4net_b200 import synth  # noqa: E402
from tests import emu  # noqa: E402

CSRC = os.path.join(ROOT, "lz4net_b200", "csrc")
# the order of enum EncProfSlot
EVENTS = ["blocks", "seqs", "rounds", "rounds_wide", "exact", "probes", "probe_hits", "flushes", "long_lit", "catchup_long"]
PHASES = ["loadhash", "samehash", "vote", "exact", "probe", "catchup", "count", "park", "emit", "block"]
BLOCK = 65536


def _build(tmp: str, prof: bool) -> C.CDLL:
    so = os.path.join(tmp, f"enc_phases_gpu_{int(prof)}.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-shared", "-Xcompiler",
                           "-fPIC", "-I" + CSRC, "-o", so, os.path.join(ROOT, "tools", "enc_phases.cu")]
                          + (["-DLZ4B200_ENC_PROF"] if prof else []))
    return C.CDLL(so)


def _per_seq(rows: np.ndarray) -> dict:
    ev = {k: int(v) for k, v in zip(EVENTS, rows[:len(EVENTS)])}
    cyc = rows[len(EVENTS):].astype(np.float64)
    seqs = max(ev["seqs"], 1)
    out = {"events": ev, "per_seq": {k: round(ev[k] / seqs, 4) for k in EVENTS if k not in ("seqs",)}}
    out["exact_rate"] = round(ev["exact"] / max(ev["rounds"], 1), 4)
    if cyc.any():
        body = cyc[:-1].sum()
        out["cycles_per_seq"] = {k: round(c / seqs, 1) for k, c in zip(PHASES, cyc)}
        out["phase_share"] = {k: round(c / body, 4) for k, c in zip(PHASES[:-1], cyc[:-1])}
        out["unattributed_share"] = round(1.0 - body / cyc[-1], 4)      # table clear and the code between laps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=None)
    ap.add_argument("--cls", default="E50,ETEXT")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--emu", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    nb = a.blocks or (8 if a.emu else 32768)
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        if a.emu:
            libs = {True: C.CDLL(emu.build(os.path.join(ROOT, "tools", "enc_phases_emu.cpp"), ["-DLZ4B200_ENC_PROF"]))}
        else:
            libs = {True: _build(tmp, True), False: _build(tmp, False)}
            import torch
            res["device"] = torch.cuda.get_device_name(0)
            try:
                res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                                    capture_output=True, text=True).stdout.strip()
            except OSError:
                pass
        for cls in a.cls.split(","):
            blocks = np.ascontiguousarray(synth.make_blocks(cls, nb, BLOCK, seed=2))
            lens = np.zeros(nb, np.int32)
            rows = np.zeros(len(EVENTS) + len(PHASES), np.uint64)
            src = C.c_void_p(blocks.ctypes.data)
            if a.emu:
                libs[True].enc_phases_emu_run(src, BLOCK, nb, C.c_void_p(lens.ctypes.data), C.c_void_p(rows.ctypes.data))
                r = _per_seq(rows)
            else:
                ms = {}
                for prof in (False, True):
                    t = C.c_float(0)
                    err = libs[prof].enc_phases_run(src, BLOCK, nb, a.reps, C.c_void_p(lens.ctypes.data),
                                                    C.c_void_p(rows.ctypes.data), C.byref(t))
                    if err:
                        raise RuntimeError(f"CUDA error {err}")
                    ms[prof] = t.value
                r = _per_seq(rows // np.uint64(a.reps))
                r["kernel_ms"] = {"plain": round(ms[False], 3), "instrumented": round(ms[True], 3)}
                r["encode_gbs_plain"] = round(nb * BLOCK / ms[False] / 1e6, 2)
            r["blocks"] = nb
            r["compressed_bytes"] = int(lens.astype(np.int64).sum())
            res[cls] = r
            print(cls, json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
