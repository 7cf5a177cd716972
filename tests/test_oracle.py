"""CPU-only: pins the port oracle (oracle/lz4_oracle.c) to the reference's own sources and to the committed golden
vectors.  Mirrors src/LZ4.Tests/ConformanceTests.cs (all encoders byte-identical, all decoders round-trip) and
original/fuzzer.c:146-233 (size +-1 invariants).  What the reference (oracle/_ref) returned on these inputs is stored in
tests/golden/reference_v1.json (tests/golden/make_golden.py): the records below are computed with the port and compared
with the reference's."""
import hashlib
import json
import os

import numpy as np
import pytest

import oracle
from tests import cases

GOLD = os.path.join(os.path.dirname(__file__), "golden", "golden_v1.json")
REF = os.path.join(os.path.dirname(__file__), "golden", "reference_v1.json")
CONSTRUCTED = os.path.join(os.path.dirname(__file__), "golden", "constructed_v1.json")
CONSTRUCTED_SEED = 1                                 # tests/lz4seq.py's corpus(seed) that constructed_v1.json records
HC_CONSTRUCTED = os.path.join(os.path.dirname(__file__), "golden", "hc_constructed_v1.json")
HC_CONSTRUCTED_SEED = 1                              # tests/hcedge.py's catalogue(seed) that hc_constructed_v1.json records


def _sha(b: bytes) -> str:
    return hashlib.sha256(b).hexdigest()


def _digest(*parts) -> str:
    h = hashlib.sha256()
    for p in parts:
        h.update(p if isinstance(p, bytes) else str(p).encode())
        h.update(b"|")
    return h.hexdigest()[:12]


def _stored(key):
    return json.load(open(REF))[key]


def records_random_lengths(model, impl):
    """[n, ret fast, ret HC, digest of every return value and output, limited outputs included] per input."""
    out = []
    lens = cases.random_lengths(60, 200_000, seed=7) + list(cases.BOUNDARY_LENGTHS)
    for i, n in enumerate(lens):
        if model in ("mixed",) and n > 70_000:
            n = n % 70_000
        data = cases.content(model, n, seed=i).tobytes()
        rets, parts = [], []
        for fn in (oracle.encode, oracle.encode_hc):
            r, o = fn(data, impl=impl)
            rets.append(r); parts += [r, o]
            # limited output: exactly enough, one short, and cap = n (fuzzer.c:212-227; LZ4Stream.cs:243-246)
            for cap in sorted({r, r - 1, n, max(0, n - 1), r // 2}):
                if cap >= 0:
                    parts += [cap, *fn(data, cap=cap, impl=impl)]
        out.append([n, *rets, _digest(*parts)])
    return out


def records_accept_reject(impl):
    """fuzzer.c:176-210 on 48 inputs: the compressed stream, known-size verdicts for n, n-1, n+1, and unknown-size verdicts
    (+ output digest) for the (input size, output capacity) pairs of _ACCEPT_REJECT_SIZES."""
    rng = np.random.default_rng(3)
    from lz4net_b200 import synth
    out = []
    for i in range(48):
        fuz = i % 6 == 5      # the upstream generator: for it the +-1 invariants are strict (fuzzer.c:176-210)
        data = (synth.fuz_block(i, 4096) if fuz else
                cases.content(cases.MODELS[i % len(cases.MODELS)], int(rng.integers(20, 40000)), seed=100 + i)).tobytes()
        n = len(data)
        _, comp = oracle.encode(data, impl=impl)
        clen = len(comp)
        known = [oracle.decode_known(comp, osize, impl=impl)[0] for osize in (n, n - 1, n + 1)]
        unknown = []
        for isz, osz in ((clen, n + 1), (clen, n), (clen, n - 1), (clen - 1, n), (clen + 1, n)):
            cc = comp if isz <= clen else comp + b"\x00"
            r, o = oracle.decode_unknown(cc[:isz], osz, impl=impl)
            unknown.append([r, _digest(o) if r >= 0 else None])
        out.append({"n": n, "fuz": fuz, "clen": clen, "comp": _digest(comp), "known": known, "unknown": unknown})
    return out


def digest_accept_reject(records):
    """What the port must share with the reference: every input, stream and verdict, and the value and output of every
    accepted decode (the magnitude of an error result is not part of parity)."""
    return _digest(*(json.dumps([r["n"], r["clen"], r["comp"], [max(a, -1) for a in r["known"]],
                                 [[max(a, -1), d] for a, d in r["unknown"]]]) for r in records))


def records_corrupt_streams(impl):
    """300 bit-flipped streams: (digest of all the streams, [unknown-size verdict, output digest or None] per stream)."""
    rng = np.random.default_rng(11)
    out, streams = [], []
    for i in range(300):
        data = cases.content("mixed", 3000, seed=i).tobytes()
        _, comp = oracle.encode(data, impl=impl)
        c = bytearray(comp)
        for _ in range(int(rng.integers(1, 4))):
            c[int(rng.integers(0, len(c)))] ^= 1 << int(rng.integers(0, 8))
        r, o = oracle.decode_unknown(bytes(c), len(data), impl=impl)
        streams.append(bytes(c)); out.append([max(r, -1), _digest(o)[:8] if r >= 0 else None])
    return _digest(*streams), out


def records_constructed(impl):
    """tests/lz4seq.py's corpus: (digest of every case's name, stream and cap, [known-size result, unknown-size result,
    output digest] per case).  Results of a rejected stream are -1.  A known-size result past the end of the stream is
    kept as it is -- the reference's LZ4_uncompress reads as far as the stream's tokens say, unbounded by design -- and
    the bytes it decoded that way are not part of the digest."""
    from tests import lz4seq
    corpus = lz4seq.corpus(CONSTRUCTED_SEED)
    rows = []
    for c in corpus:
        rk, ok = oracle.decode_known(c.stream, c.cap, impl=impl)
        ru, ou = oracle.decode_unknown(c.stream, c.cap, impl=impl)
        rows.append([max(rk, -1), max(ru, -1),
                     _digest(ok if 0 <= rk <= len(c.stream) else b"-", ou if ru >= 0 else b"-")[:8]])
    return _digest(*(p for c in corpus for p in (c.name, c.stream, c.cap))), rows


def records_hc_constructed(corpus, impl):
    """tests/hcedge.py's blocks: [name, ret, digest, ret and digest at cap = n, at cap = ret - 1] per case (the last
    pair only where ret > 0)."""
    rows = []
    for c in corpus:
        r, o = oracle.encode_hc(c.data, impl=impl)
        row = [c.name, r, _sha(o)]
        for cap in (len(c.data), r - 1):
            if cap >= 0:
                rc, oc = oracle.encode_hc(c.data, cap=cap, impl=impl)
                row += [rc, _sha(oc)]
        rows.append(row)
    return rows


def test_bound():
    for n in (0, 1, 254, 255, 256, 65536, 1 << 20):
        assert oracle.bound(n) == oracle.port().lz4o_bound(n) == n + n // 255 + 16
    assert oracle.bound(65536) == 65809            # src/LZ4/LZ4Codec.cs:313-316


def test_golden_vectors_port():
    """The port reproduces every committed golden vector (made from oracle/_ref by make_golden.py)."""
    g = json.load(open(GOLD))
    assert len(g["cases"]) >= 40
    for c in g["cases"]:
        data = cases.AUTOTEST if c["model"] == "autotest" else cases.content(c["model"], c["n"], c["seed"]).tobytes()
        assert _sha(data) == c["input_sha256"], c["name"]
        for mode, fn in (("fast", oracle.encode), ("hc", oracle.encode_hc)):
            r, out = fn(data, impl="port")
            assert r == c[mode]["len"], (c["name"], mode)
            assert _sha(out) == c[mode]["sha256"], (c["name"], mode)
            if "hex" in c[mode]:
                assert out.hex() == c[mode]["hex"]
            rr, dec = oracle.decode_known(out, len(data), impl="port")
            assert rr == r and dec == data
            # LZ4Stream / Wrap pass cap = n (src/LZ4/LZ4Stream.cs:243-246): the stored-raw decision is part of parity
            r2, _ = fn(data, cap=len(data), impl="port")
            assert r2 == c[mode]["len_cap_n"], (c["name"], mode)


@pytest.mark.parametrize("model", cases.MODELS)
def test_port_equals_reference_random_lengths(model):
    got = records_random_lengths(model, "port")
    assert _digest(*got) == _stored("random_lengths")[model], model
    for i, (n, _, _, _) in enumerate(got):
        data = cases.content(model, n, seed=i).tobytes()
        r, o = oracle.encode(data)
        d1 = oracle.decode_known(o, n, impl="port")
        d2 = oracle.decode_unknown(o, n, impl="port")
        assert d1 == (r, data) and d2 == (n if n else d2[0], data)


def test_decoders_accept_reject_like_reference():
    """fuzzer.c:176-210: exact size works, size +-1 must fail; the port takes the same decisions as the reference."""
    got = records_accept_reject("port")
    assert digest_accept_reject(got) == _stored("accept_reject")          # the same decisions as the reference
    for g in got:
        n, clen = g["n"], g["clen"]
        for osize, a in zip((n, n - 1, n + 1), g["known"]):
            assert (osize == n) == (a >= 0)
        sizes = ((clen, n + 1), (clen, n), (clen, n - 1), (clen - 1, n), (clen + 1, n))
        for (isz, osz), a in zip(sizes, g["unknown"]):
            if g["fuz"] or isz == clen:
                # (on arbitrary data a truncated stream can, rarely, still parse: the match-length loop stops at
                #  iend-6 and re-reads its last byte as a token, original/lz4.c:986-999)
                assert (a[0] >= 0) == (isz == clen and osz >= n)


def test_corrupt_streams_same_verdict():
    """Bit-flipped streams: the port must never crash and must agree with the reference on accept/reject
    (and on the bytes when both accept), except for offset-0 matches which the port rejects by design."""
    agree = 0
    (want_streams, want), (got_streams, got) = _stored("corrupt_streams"), records_corrupt_streams("port")
    assert got_streams == want_streams                 # the same corrupted streams
    for a, b in zip(want, got):
        if (a[0] < 0) == (b[0] < 0):
            agree += 1
            if a[0] >= 0:
                assert a == b
        else:
            assert a[0] >= 0 and b[0] < 0          # only the documented tightening (offset == 0)
    assert agree >= 290


def test_fuz_generator_roundtrip():
    from lz4net_b200 import synth
    for seed in range(4):
        data = synth.fuz_block(seed, 8192).tobytes()
        r, c = oracle.encode(data)
        rh, ch = oracle.encode_hc(data)
        assert oracle.decode_known(c, len(data)) == (r, data)
        assert oracle.decode_known(ch, len(data)) == (rh, data)
        assert oracle.decode_known(c, len(data) - 1)[0] < 0 and oracle.decode_known(c, len(data) + 1)[0] < 0


def test_mt_run_port_matches_single_calls():
    """bench.py's CPU baseline times the port through oracle.mt_run when oracle/_ref is absent (a default build)."""
    from lz4net_b200 import synth
    n, bs = 12, 65536
    raw = synth.make_blocks("E50", n, bs, seed=5).reshape(-1)
    slot = oracle.bound(bs)
    so = np.arange(n, dtype=np.int64) * bs; do = np.arange(n, dtype=np.int64) * slot
    sl = np.full(n, bs, np.int32); dc = np.full(n, slot, np.int32)
    for kind, fn in (("encode", oracle.encode), ("encode_hc", oracle.encode_hc)):
        comp = np.zeros(n * slot + 64, np.uint8)
        _, clen = oracle.mt_run(kind, "port", raw, so, sl, comp, do, dc, 3)
        for i in range(n):
            r, o = fn(raw[i * bs:(i + 1) * bs])
            assert clen[i] == r and comp[do[i]:do[i] + r].tobytes() == o, (kind, i)
        out = np.zeros(n * bs + 64, np.uint8)
        _, used = oracle.mt_run("decode", "port", comp, do, clen, out, so, sl, 3)
        assert np.array_equal(used, clen) and np.array_equal(out[:n * bs], raw), kind


def test_port_equals_reference_on_constructed_streams():
    """tests/lz4seq.py's constructed streams -- every end-of-block rule, offset and length threshold at the exact byte,
    truncated, extended and under shifted caps: the port returns what the reference returned (constructed_v1.json, made
    by make_golden.py), with the two documented exceptions:
    * offset 0: the port rejects it (the reference copies output bytes nobody has written yet);
    * a known-size decode the reference accepts only by reading past the end of the stream: the port, like every decoder
      of this project, reads nothing outside [src, src + isize) and rejects it."""
    from tests import lz4seq
    stored = json.load(open(CONSTRUCTED))
    want = stored["cases"]
    assert _digest(*(json.dumps(w) for w in want)) == stored["rows"], "constructed_v1.json differs from what make_golden.py wrote"
    corpus = lz4seq.corpus(CONSTRUCTED_SEED)
    digest, got = records_constructed("port")
    assert digest == stored["corpus"], "tests/lz4seq.py no longer makes the corpus the fixture was made from"
    offset0 = 0
    for c, w, g in zip(corpus, want, got):
        if "/off0/" in c.name:
            assert g[:2] == [-1, -1], c.name
            offset0 += w[0] >= 0 or w[1] >= 0
        elif w[0] > len(c.stream):
            assert g[0] == -1 and g[1:] == w[1:], c.name
        else:
            assert g == w, (c.name, g, w)
    past = sum(w[0] > len(c.stream) for c, w in zip(corpus, want))
    assert offset0 > 0 and past == stored["known_reads_past_isize"] > 0


def test_port_equals_reference_on_constructed_hc_blocks():
    """tests/hcedge.py's blocks -- candidates at the ends of the attempt budget, position 0, ties, lengths at matchlimit
    and around the warp count's steps, backward extensions, repeats, the 64 KiB window: the port's LZ4HC returns what the
    reference returned (hc_constructed_v1.json, made by make_golden.py), uncapped and at the two capacities LZ4Stream and
    a one-byte shortfall give."""
    from tests import hcedge
    stored = json.load(open(HC_CONSTRUCTED))
    corpus = hcedge.catalogue(HC_CONSTRUCTED_SEED)
    assert _digest(*(p for c in corpus for p in (c.name, c.data))) == stored["corpus"], \
        "tests/hcedge.py no longer makes the blocks the fixture was made from"
    got = records_hc_constructed(corpus, "port")
    assert len(got) == len(stored["cases"])
    for g, w in zip(got, stored["cases"]):
        assert g == w, g[0]
