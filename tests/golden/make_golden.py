"""Regenerates tests/golden/golden_v1.json and tests/golden/reference_v1.json from the REFERENCE's own code
(oracle/_ref/liblz4net_ref.so, i.e. a lz4net checkout's original/lz4.c + lz4hc.c compiled in place by oracle/Makefile):

    LZ4NET_REFERENCE=<lz4net checkout> python tests/golden/make_golden.py

golden_v1.json: encoder outputs on named inputs.  reference_v1.json: the reference's side of tests/test_oracle.py's
port-versus-reference checks (return values and output digests), and the one input on which r93's LZ4HC gives up at
LZ4_compressBound (tests/test_kernels_emu.py).  constructed_v1.json: what both reference decoders return on the
constructed streams of tests/lz4seq.py, one case per line.  hc_constructed_v1.json: what the reference's LZ4HC returns
on the constructed blocks of tests/hcedge.py, uncapped, at cap = n and at cap = ret - 1, one case per line.

The reference ships no golden vectors of its own (SURVEY.md 8c); these are outputs of the reference itself on
reproducible inputs (tests/cases.py), including the reference-defined AutoTest text (src/LZ4/LZ4Codec.cs:175-184).
"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402
from tests import cases, hcedge, lz4seq  # noqa: E402


def sha(b):
    return hashlib.sha256(b).hexdigest()


def main():
    out = []
    todo = [("autotest", "autotest", len(cases.AUTOTEST), 0)]
    for m in cases.MODELS:
        todo.append((f"{m}-64k", m, 65536, 1))
    for i, n in enumerate((0, 1, 12, 13, 20, 64, 300, 4096, 32768, 65535, 65546, 65547, 100000)):
        for m in ("mixed", "lowent", "ETEXT", "periodic"):
            todo.append((f"{m}-{n}", m, n if not (m == 'mixed' and n > 70000) else 70000, 50 + i))
    seen = set()
    for name, model, n, seed in todo:
        if name in seen:
            continue
        seen.add(name)
        data = cases.AUTOTEST if model == "autotest" else cases.content(model, n, seed).tobytes()
        c = {"name": name, "model": model, "n": len(data), "seed": seed, "input_sha256": sha(data)}
        for mode, fn in (("fast", oracle.encode), ("hc", oracle.encode_hc)):
            r, o = fn(data, impl="ref")
            r2, _ = fn(data, cap=len(data), impl="ref")
            c[mode] = {"len": r, "sha256": sha(o), "len_cap_n": r2}
            if r <= 512:
                c[mode]["hex"] = o.hex()
        out.append(c)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden_v1.json")
    json.dump({"source": "oracle/_ref (reference original/lz4.c + lz4hc.c, LZ4_ARCH64=1, LZ4_MK_OPT)", "cases": out},
              open(path, "w"), indent=1)
    print("wrote", path, len(out), "cases")

    from lz4net_b200 import synth
    from tests import test_oracle as t
    d = synth.make_blocks("E0", 1, 65536, seed=3, first_block=1268)[0].tobytes()
    ref = {"source": "oracle/_ref (reference original/lz4.c + lz4hc.c, LZ4_ARCH64=1, LZ4_MK_OPT)",
           "random_lengths": {m: t._digest(*t.records_random_lengths(m, "ref")) for m in cases.MODELS},
           "accept_reject": t.digest_accept_reject(t.records_accept_reject("ref")),
           "corrupt_streams": t.records_corrupt_streams("ref"),
           "hc_gives_up_at_bound": {"class": "E0", "seed": 3, "first_block": 1268,
                                    "ret": oracle.encode_hc(d, cap=oracle.bound(len(d)), impl="ref")[0]}}
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_v1.json")
    with open(path, "w") as f:
        json.dump(ref, f, separators=(",", ":"))
        f.write("\n")
    print("wrote", path)

    digest, rows = t.records_constructed("ref")
    past = sum(r[0] > len(c.stream) for c, r in zip(lz4seq.corpus(t.CONSTRUCTED_SEED), rows))
    head = {"source": ref["source"], "generator": "tests/lz4seq.py", "seed": t.CONSTRUCTED_SEED, "corpus": digest,
            "rows": t._digest(*(json.dumps(r) for r in rows)), "known_reads_past_isize": past,
            "row": "[known-size result, unknown-size result, output digest]; -1 = rejected; a known-size result above the "
                   "stream's length = accepted by reading past isize"}
    with open(t.CONSTRUCTED, "w") as f:
        f.write(json.dumps(head, separators=(",", ":"))[:-1] + ',"cases":[\n')
        f.write(",\n".join(json.dumps(r, separators=(",", ":")) for r in rows))
        f.write("\n]}\n")
    print("wrote", t.CONSTRUCTED, len(rows), "cases,", past, "known-size decodes accepted only by reading past isize")

    corpus = hcedge.catalogue(t.HC_CONSTRUCTED_SEED)
    rows = t.records_hc_constructed(corpus, "ref")
    head = {"source": ref["source"], "generator": "tests/hcedge.py", "seed": t.HC_CONSTRUCTED_SEED,
            "corpus": t._digest(*(p for c in corpus for p in (c.name, c.data))),
            "row": "[name, ret, sha256, ret at cap = n, sha256, ret at cap = ret - 1 (absent when ret = 0), sha256]"}
    with open(t.HC_CONSTRUCTED, "w") as f:
        f.write(json.dumps(head, separators=(",", ":"))[:-1] + ',"cases":[\n')
        f.write(",\n".join(json.dumps(r, separators=(",", ":")) for r in rows))
        f.write("\n]}\n")
    print("wrote", t.HC_CONSTRUCTED, len(rows), "cases")


if __name__ == "__main__":
    main()
