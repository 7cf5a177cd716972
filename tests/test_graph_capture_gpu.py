"""CUDA graphs of the device-memory calls, on an H100.

Every device-memory entry point is captured once on a fresh context (after lz4b200_reserve, with no eager call on that
context first) and replayed with new contents in its static input tensors: a different entropy class each time, and for
the decoders and Unwrap a batch with malformed blocks or packets.  Each replay must give what the same call gives eagerly
on a second context.  Then: a chain of calls in one graph, replays interleaved with eager calls on the shared scratch,
graphs that keep their block counters while eager calls go round the ring, growth of the scratch after a capture, the
refusal of a capture the scratch was not reserved for and of the synchronous calls, and the memory a context that never
captured keeps."""
import numpy as np
import pytest

import oracle
from lz4net_b200 import synth

pytestmark = pytest.mark.gpu

E_ARG = -1
GUARD = 0xA5


def _torch():
    import torch
    return torch


def _ctx():
    from lz4net_b200.codec import Context
    return Context(0)


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a)).cuda()


def _blocks(cls, n, size, seed=5):
    return synth.make_blocks(cls, n, size, seed=seed)


def _uniform(n, stride, length):
    return _dev(np.arange(n, dtype=np.int64) * stride), _dev(np.full(n, length, np.int32))


def _load(t, feed):
    for k, v in feed.items():
        t[k].copy_(v if isinstance(v, _torch().Tensor) else _dev(v))


def _clear(t, outs):
    for k in outs:
        t[k].fill_(GUARD) if t[k].dtype == _torch().uint8 else t[k].fill_(-7)


def _capture(ctx, call, t, stream=None):
    torch = _torch()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        call(ctx, t)
    return g


def _same(got, want, outs, compare):
    torch = _torch()
    if compare is not None:
        compare(got, want)
        return
    for k in outs:
        assert torch.equal(got[k], want[k]), k


def _check_replays(call, t, outs, feeds, reserve, compare=None):
    """Capture call(ctx, t) on a fresh reserved context with feeds[0] loaded, then replay it once per feed; each replay's
    output tensors, whole, equal an eager call's on a second context, both starting from the same guard-filled outputs
    (the bytes an encoder leaves behind out_len and a rejected block's partial output included)."""
    torch = _torch()
    ctx, ref = _ctx(), _ctx()
    try:
        ctx.reserve(*reserve)
        _load(t, feeds[0])
        _clear(t, outs)
        torch.cuda.synchronize()
        before = ctx.launches
        g = _capture(ctx, call, t)
        assert ctx.launches > before or not outs                       # counted at capture
        for feed in feeds[1:] + feeds[:1]:
            _load(t, feed)
            _clear(t, outs)
            want = {k: v.clone() for k, v in t.items()}
            g.replay()
            call(ref, want)
            torch.cuda.synchronize()
            _same(t, want, outs, compare)
        del g
    finally:
        torch.cuda.synchronize()
        ctx.close()
        ref.close()


# ---- inputs ----------------------------------------------------------------------------------------------------------
def _encode_tensors(n, size):
    torch = _torch()
    slot = oracle.bound(size)
    so, sl = _uniform(n, size, size)
    do, dc = _uniform(n, slot, slot)
    return dict(raw=torch.zeros(n * size, dtype=torch.uint8, device="cuda"), so=so, sl=sl,
                slots=torch.zeros(n * slot, dtype=torch.uint8, device="cuda"), do=do, dc=dc,
                out=torch.zeros(n, dtype=torch.int32, device="cuda"))


def _comp_feed(cls, n, size, slot, hc=False, malformed=False, seed=5):
    """Compressed blocks of one class in fixed slots; malformed: a truncated block, a corrupted one, a bad offset."""
    raws = _blocks(cls, n, size, seed)
    comp = np.zeros(n * slot, np.uint8)
    lens = np.zeros(n, np.int32)
    for i in range(n):
        r, o = (oracle.encode_hc if hc else oracle.encode)(raws[i].tobytes())
        comp[i * slot:i * slot + r] = np.frombuffer(o, np.uint8)
        lens[i] = r
    if malformed:
        lens[0] = max(lens[0] - 5, 1)                                   # truncated
        comp[slot + 1:slot + 9] = 0xFF                                  # long literal run past the end
        comp[2 * slot + lens[2] - 8:2 * slot + lens[2] - 6] = 0xFF      # an offset near the end
        lens[3] = 0                                                     # empty input
    return dict(comp=comp, sl=lens)


def _decode_tensors(n, size):
    torch = _torch()
    slot = oracle.bound(size)
    so, _ = _uniform(n, slot, 0)
    do, dc = _uniform(n, size, size)
    return slot, dict(comp=torch.zeros(n * slot, dtype=torch.uint8, device="cuda"), so=so,
                      sl=torch.zeros(n, dtype=torch.int32, device="cuda"),
                      dst=torch.zeros(n * size, dtype=torch.uint8, device="cuda"), do=do, dc=dc,
                      out=torch.zeros(n, dtype=torch.int32, device="cuda"))


def _decode_feeds(n, size, slot):
    return [_comp_feed("E100", n, size, slot), _comp_feed("E50", n, size, slot, hc=True), _comp_feed("ETEXT", n, size, slot),
            _comp_feed("ETEXT", n, size, slot, malformed=True, seed=9)]


def _packets(inputs, hc):
    from lz4net_b200.codec import wrap_batch
    ctx = _ctx()
    try:
        return wrap_batch(inputs, hc=hc, ctx=ctx)
    finally:
        ctx.close()


def _packet_feed(cls, n, size, pslot, hc=False, malformed=False, seed=5):
    pk = _packets([b.tobytes() for b in _blocks(cls, n, size, seed)], hc)
    buf = np.zeros(n * pslot, np.uint8)
    lens = np.zeros(n, np.int32)
    for i, p in enumerate(pk):
        buf[i * pslot:i * pslot + len(p)] = np.frombuffer(p, np.uint8)
        lens[i] = len(p)
    if malformed:
        buf[0:4] = np.frombuffer((size * 4).to_bytes(4, "little"), np.uint8)       # above its capacity: E_ARG
        lens[1] = 5                                                                 # shorter than a header: E_FORMAT
        buf[2 * pslot + 4:2 * pslot + 8] = np.frombuffer((size * 2).to_bytes(4, "little"), np.uint8)   # stored > packet
        if lens[3] > 20:
            buf[3 * pslot + 12:3 * pslot + 16] = 0xFF                               # a corrupted payload
    return dict(pk=buf, sl=lens)


def _unwrap_tensors(n, size):
    torch = _torch()
    pslot = size + 8
    so, _ = _uniform(n, pslot, 0)
    do, dc = _uniform(n, size, size)
    return pslot, dict(pk=torch.zeros(n * pslot, dtype=torch.uint8, device="cuda"), so=so,
                       sl=torch.zeros(n, dtype=torch.int32, device="cuda"),
                       dst=torch.zeros(n * size, dtype=torch.uint8, device="cuda"), do=do, dc=dc,
                       off=torch.zeros(n + 1, dtype=torch.int64, device="cuda"),
                       out=torch.zeros(n, dtype=torch.int32, device="cuda"))


def _unwrap_feeds(n, size, pslot):
    return [_packet_feed("E100", n, size, pslot), _packet_feed("E0", n, size, pslot), _packet_feed("E50", n, size, pslot, hc=True),
            _packet_feed("ETEXT", n, size, pslot, malformed=True, seed=9)]


# ---- 1. every entry point --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hc,n,size", [(False, 48, 4096), (True, 24, 16384), (True, 4, 80000)],
                         ids=["fast", "hc-small-blocks", "hc-blocks-above-64k"])
def test_capture_encode(hc, n, size):
    from lz4net_b200 import batch
    t = _encode_tensors(n, size)
    feeds = [dict(raw=_blocks(c, n, size).reshape(-1)) for c in ("E100", "E0", "E50", "ETEXT")]
    _check_replays(lambda ctx, t: batch.encode(ctx, t["raw"], t["so"], t["sl"], t["slots"], t["do"], t["dc"], t["out"], hc=hc),
                   t, ["slots", "out"], feeds, (n, hc))


@pytest.mark.parametrize("lanes", [0, 16, 1], ids=["auto", "lanes16", "lane-per-block"])
@pytest.mark.parametrize("known", [True, False], ids=["known", "unknown"])
def test_capture_decode(known, lanes):
    from lz4net_b200 import batch
    n, size = 40, 4096
    slot, t = _decode_tensors(n, size)

    def call(ctx, t):
        if lanes:
            ctx.set_option("decode_lanes", lanes)
        batch.decode(ctx, t["comp"], t["so"], t["sl"], t["dst"], t["do"], t["dc"], t["out"], known=known)
    _check_replays(call, t, ["dst", "out"], _decode_feeds(n, size, slot), (n, False))


@pytest.mark.parametrize("known", [True, False], ids=["known", "unknown"])
def test_capture_measure(known):
    from lz4net_b200 import batch
    n, size = 40, 4096
    slot, t = _decode_tensors(n, size)
    _check_replays(lambda ctx, t: batch.measure(ctx, t["comp"], t["so"], t["sl"], t["out"], t["dc"] if known else None, known=known),
                   t, ["out"], _decode_feeds(n, size, slot), (n, False))


@pytest.mark.parametrize("fits", [True, False], ids=["fits", "does-not-fit"])
def test_capture_decode_packed(fits):
    from lz4net_b200 import batch
    torch = _torch()
    n, size = 40, 4096
    slot, t = _decode_tensors(n, size)
    t["dst"] = torch.zeros(n * size if fits else size, dtype=torch.uint8, device="cuda")
    t["off"] = torch.zeros(n + 1, dtype=torch.int64, device="cuda")

    def compare(got, want):
        for k in ("dst", "off", "out"):
            assert torch.equal(got[k], want[k]), k
        assert fits or (got["dst"] == GUARD).all()                        # too small: untouched
    _check_replays(lambda ctx, t: batch.decode_packed(ctx, t["comp"], t["so"], t["sl"], t["dst"], t["off"], t["out"]),
                   t, ["dst", "off", "out"], _decode_feeds(n, size, slot), (n, False), compare)


def test_capture_compact():
    from lz4net_b200 import batch
    torch = _torch()
    n, size = 300, 2048
    slot, t = _decode_tensors(n, size)
    t["packed"] = torch.zeros(n * slot, dtype=torch.uint8, device="cuda")
    t["off"] = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    feeds = [f for f in _decode_feeds(n, size, slot)]
    feeds[-1]["sl"][5] = -3                                              # a failed block occupies no bytes
    _check_replays(lambda ctx, t: batch.compact(ctx, t["comp"], t["so"], t["sl"], t["packed"], t["off"]),
                   t, ["packed", "off"], feeds, (n, False))


@pytest.mark.parametrize("hc", [False, True], ids=["fast", "hc"])
def test_capture_wrap_device(hc):
    from lz4net_b200 import batch
    torch = _torch()
    n, size = 32, 8192
    so, sl = _uniform(n, size, size)
    do, dc = _uniform(n, size + 8, size + 8)
    t = dict(raw=torch.zeros(n * size, dtype=torch.uint8, device="cuda"), so=so, sl=sl,
             pk=torch.zeros(n * (size + 8), dtype=torch.uint8, device="cuda"), do=do, dc=dc,
             out=torch.zeros(n, dtype=torch.int32, device="cuda"))
    feeds = [dict(raw=_blocks(c, n, size).reshape(-1)) for c in ("E100", "E0", "E50", "ETEXT")]
    _check_replays(lambda ctx, t: batch.wrap(ctx, t["raw"], t["so"], t["sl"], t["pk"], t["do"], t["dc"], t["out"], hc=hc),
                   t, ["pk", "out"], feeds, (n, hc))


def test_capture_unwrap_device():
    from lz4net_b200 import batch
    n, size = 32, 8192
    pslot, t = _unwrap_tensors(n, size)
    _check_replays(lambda ctx, t: batch.unwrap(ctx, t["pk"], t["so"], t["sl"], t["dst"], t["do"], t["dc"], t["out"]),
                   t, ["dst", "out"], _unwrap_feeds(n, size, pslot), (n, False))


def test_capture_unwrap_packed():
    from lz4net_b200 import batch
    n, size = 32, 8192
    pslot, t = _unwrap_tensors(n, size)
    _check_replays(lambda ctx, t: batch.unwrap_packed(ctx, t["pk"], t["so"], t["sl"], t["dst"], t["off"], t["out"]),
                   t, ["dst", "off", "out"], _unwrap_feeds(n, size, pslot), (n, False))


def test_capture_synth_fill():
    from lz4net_b200 import batch
    torch = _torch()
    n, size = 16, 4096
    t = dict(dst=torch.zeros(n * size, dtype=torch.uint8, device="cuda"))
    for cls in range(4):
        _check_replays(lambda ctx, t: batch.synth_fill(ctx, t["dst"], n, size, cls, seed=3), t, ["dst"], [{}, {}, {}], (0, False))
        assert t["dst"].cpu().numpy().tobytes() == synth.make_blocks(synth.CLASSES[cls], n, size, seed=3).tobytes()


# ---- 2. a chain in one graph -----------------------------------------------------------------------------------------
def test_capture_encode_compact_decode_packed_chain():
    from lz4net_b200 import batch
    torch = _torch()
    n, size = 64, 8192
    t = _encode_tensors(n, size)
    t["packed"] = torch.zeros(n * oracle.bound(size), dtype=torch.uint8, device="cuda")
    t["off"] = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    t["back"] = torch.zeros(n * size, dtype=torch.uint8, device="cuda")
    t["boff"] = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    t["bout"] = torch.zeros(n, dtype=torch.int32, device="cuda")

    def chain(ctx, t):
        batch.encode(ctx, t["raw"], t["so"], t["sl"], t["slots"], t["do"], t["dc"], t["out"])
        batch.compact(ctx, t["slots"], t["do"], t["out"], t["packed"], t["off"])
        batch.decode_packed(ctx, t["packed"], t["off"][:n], t["out"], t["back"], t["boff"], t["bout"])   # n block offsets
    ctx = _ctx()
    try:
        ctx.reserve(n)
        g = _capture(ctx, chain, t)
        for cls in ("E0", "E50", "ETEXT", "E100"):
            raws = _blocks(cls, n, size, seed=21)
            t["raw"].copy_(_dev(raws.reshape(-1)))
            t["back"].fill_(GUARD)
            g.replay()
            torch.cuda.synchronize()
            comp = [oracle.encode(b.tobytes())[1] for b in raws]
            assert t["out"].tolist() == [len(c) for c in comp], cls
            assert t["packed"][:int(t["off"][n])].cpu().numpy().tobytes() == b"".join(comp), cls
            assert t["back"].cpu().numpy().tobytes() == raws.tobytes(), cls
            assert t["bout"].tolist() == [size] * n and t["boff"].tolist() == list(range(0, n * size + 1, size)), cls
        del g
    finally:
        torch.cuda.synchronize()
        ctx.close()


# ---- 3. replays interleaved with eager calls on the shared scratch ---------------------------------------------------
def _interleave(make, reserve_n, hc):
    """make(seed) -> (tensors, call, check): two batches of one kind on one context, one captured and replayed on stream A,
    one enqueued eagerly on stream B right behind (and in front of) the replay, with no synchronise in between."""
    torch = _torch()
    ctx = _ctx()
    try:
        ctx.reserve(reserve_n, hc)
        ta, call, check_a = make(31)
        tb, _, check_b = make(47)
        a, b = torch.cuda.Stream(), torch.cuda.Stream()
        torch.cuda.synchronize()
        g = _capture(ctx, call, ta, stream=a)
        for order in ("replay-first", "eager-first", "replay-first"):
            for t in (ta, tb):
                for k in t.get("outs", ()):
                    t[k].fill_(GUARD)
            torch.cuda.synchronize()
            for step in ((0, 1) if order == "replay-first" else (1, 0)):
                if step == 0:
                    with torch.cuda.stream(a):
                        g.replay()
                else:
                    with torch.cuda.stream(b):
                        call(ctx, tb)
            torch.cuda.synchronize()
            check_a(ta)
            check_b(tb)
        del g
    finally:
        torch.cuda.synchronize()
        ctx.close()


def test_interleave_hc_encode():
    from lz4net_b200 import batch
    n, size = 96, 16384

    def make(seed):
        t = _encode_tensors(n, size)
        raws = _blocks(("E50", "ETEXT")[seed % 2], n, size, seed)
        t["raw"].copy_(_dev(raws.reshape(-1)))
        t["outs"] = ("slots", "out")
        want = [oracle.encode_hc(b.tobytes())[1] for b in raws]

        def check(t):
            slots, slot = t["slots"].cpu().numpy(), oracle.bound(size)
            assert t["out"].tolist() == [len(w) for w in want]
            assert [slots[i * slot:i * slot + len(w)].tobytes() for i, w in enumerate(want)] == want
        return t, lambda ctx, t: batch.encode(ctx, t["raw"], t["so"], t["sl"], t["slots"], t["do"], t["dc"], t["out"], hc=True), check
    _interleave(make, n, True)


def test_interleave_compact():
    from lz4net_b200 import batch
    torch = _torch()
    n, size = 20000, 256

    def make(seed):
        rng = np.random.default_rng(seed)
        lens = rng.integers(-2, size + 1, n).astype(np.int32)
        slots = rng.integers(0, 256, n * size, dtype=np.uint8)
        t = dict(slots=_dev(slots), so=_dev(np.arange(n, dtype=np.int64) * size), sl=_dev(lens),
                 packed=torch.zeros(n * size, dtype=torch.uint8, device="cuda"),
                 off=torch.zeros(n + 1, dtype=torch.int64, device="cuda"), outs=("packed", "off"))
        keep = np.maximum(lens, 0)
        want_off = np.concatenate([[0], np.cumsum(keep)]).tolist()
        want = b"".join(slots[i * size:i * size + k].tobytes() for i, k in enumerate(keep))

        def check(t):
            assert t["off"].tolist() == want_off
            assert t["packed"][:want_off[-1]].cpu().numpy().tobytes() == want
        return t, lambda ctx, t: batch.compact(ctx, t["slots"], t["so"], t["sl"], t["packed"], t["off"]), check
    _interleave(make, n, False)


def test_interleave_unwrap_packed():
    from lz4net_b200 import batch
    n, size = 48, 32768

    def make(seed):
        pslot, t = _unwrap_tensors(n, size)
        raws = _blocks(("E50", "ETEXT")[seed % 2], n, size, seed)
        _load(t, _packet_feed(("E50", "ETEXT")[seed % 2], n, size, pslot, seed=seed))
        t["outs"] = ("dst", "off", "out")

        def check(t):
            assert t["out"].tolist() == [size] * n
            assert t["off"].tolist() == list(range(0, n * size + 1, size))
            assert t["dst"].cpu().numpy().tobytes() == raws.tobytes()
        return t, lambda ctx, t: batch.unwrap_packed(ctx, t["pk"], t["so"], t["sl"], t["dst"], t["off"], t["out"]), check
    _interleave(make, n, False)


# ---- 4. captured calls keep their block counters ---------------------------------------------------------------------
def test_graphs_keep_their_counters_while_eager_calls_go_round_the_ring():
    """Eager calls take block counters from a ring of 64 sets.  Were a captured call given a ring set, g1 and g2 (captured
    first on a fresh context) would hold sets 0 and 1 for ever.  Before each round, eager calls bring the ring round so
    that the eager encodes running next to the replays take exactly those sets, 0 and 1; the replays and those encodes
    then share a block counter unless captured calls have counters of their own, and blocks go missing on both sides."""
    from lz4net_b200 import batch
    torch = _torch()
    n, size, ring = 4096, 8192, 64
    ctx = _ctx()
    try:
        ctx.reserve(n)
        enc = lambda ctx, t: batch.encode(ctx, t["raw"], t["so"], t["sl"], t["slots"], t["do"], t["dc"], t["out"])  # noqa: E731
        batches = []
        for i, cls in enumerate(("E50", "ETEXT", "E0", "E50", "ETEXT")):
            t = _encode_tensors(n, size)
            raws = _blocks(cls, n, size, seed=60 + i)
            t["raw"].copy_(_dev(raws.reshape(-1)))
            batches.append((t, [oracle.encode(b.tobytes())[1] for b in raws]))
        g1, g2 = _capture(ctx, enc, batches[0][0]), _capture(ctx, enc, batches[1][0])
        small = _encode_tensors(4, 1024)
        small["raw"].copy_(_dev(_blocks("ETEXT", 4, 1024).reshape(-1)))
        eager = 0                                                        # eager encodes on ctx so far

        def check(t, want):
            slots, slot = t["slots"].cpu().numpy(), oracle.bound(size)
            assert t["out"].tolist() == [len(w) for w in want]
            assert [slots[i * slot:i * slot + len(w)].tobytes() for i, w in enumerate(want)] == want
        for rnd in range(3):
            # bring the ring to where the encodes on s3 take sets 0 and 1 (the graphs' sets, had they taken the ring's
            # first two); more than a whole turn the first time
            k = (-(2 + eager)) % ring + (ring if rnd == 0 else 0)
            for _ in range(k):
                enc(ctx, small)
            eager += k
            for t, _w in batches:
                t["slots"].zero_(); t["out"].zero_()
            torch.cuda.synchronize()
            s1, s2, s3 = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
            with torch.cuda.stream(s1):
                g1.replay()
            with torch.cuda.stream(s2):
                g2.replay()
            with torch.cuda.stream(s3):
                for t, _w in batches[2:]:
                    enc(ctx, t)
            eager += len(batches) - 2
            torch.cuda.synchronize()
            for t, want in batches:
                check(t, want)
        del g1, g2
    finally:
        torch.cuda.synchronize()
        ctx.close()


# ---- 5. growth after a capture ---------------------------------------------------------------------------------------
def test_replay_after_the_scratch_grew():
    """Graphs captured at reserve(n) replay correctly after eager calls on 4n blocks grew the HC arena, the scan scratch
    and the packet view, and after set_option("hc_concurrency") dropped the arena."""
    from lz4net_b200 import batch
    torch = _torch()
    ctx = _ctx()
    try:
        n_hc, hc_size = 64, 4096
        n, size = 200_000, 16                                            # the scan scratch grows in 8 bytes per 1024 blocks
        ctx.reserve(n)
        ctx.reserve(n_hc, hc=True)
        th = _encode_tensors(n_hc, hc_size)
        raws = _blocks("ETEXT", n_hc, hc_size)
        th["raw"].copy_(_dev(raws.reshape(-1)))
        want_hc = [oracle.encode_hc(b.tobytes())[1] for b in raws]
        tw = dict(raw=_dev(_blocks("E50", n, size).reshape(-1)))
        tw["so"], tw["sl"] = _uniform(n, size, size)
        tw["do"], tw["dc"] = _uniform(n, size + 8, size + 8)
        tw["pk"] = torch.zeros(n * (size + 8), dtype=torch.uint8, device="cuda")
        tw["out"] = torch.zeros(n, dtype=torch.int32, device="cuda")
        tw["packed"] = torch.zeros(n * (size + 8), dtype=torch.uint8, device="cuda")
        tw["off"] = torch.zeros(n + 1, dtype=torch.int64, device="cuda")

        def wrap_compact(ctx, t):
            batch.wrap(ctx, t["raw"], t["so"], t["sl"], t["pk"], t["do"], t["dc"], t["out"])
            batch.compact(ctx, t["pk"], t["do"], t["out"], t["packed"], t["off"])
        gh = _capture(ctx, lambda ctx, t: batch.encode(ctx, t["raw"], t["so"], t["sl"], t["slots"], t["do"], t["dc"], t["out"], hc=True), th)
        gw = _capture(ctx, wrap_compact, tw)
        gh.replay(); gw.replay()
        torch.cuda.synchronize()
        want_pk = tw["packed"][:int(tw["off"][n])].clone()
        ref = _ctx()
        try:
            rw = {k: v.clone() for k, v in tw.items()}
            wrap_compact(ref, rw)
            torch.cuda.synchronize()
            assert torch.equal(rw["packed"][:int(rw["off"][n])], want_pk)
        finally:
            ref.close()

        # eager calls on 4n blocks grow every piece
        big = _encode_tensors(4 * n_hc, hc_size)
        big["raw"].copy_(_dev(_blocks("E50", 4 * n_hc, hc_size).reshape(-1)))
        batch.encode(ctx, big["raw"], big["so"], big["sl"], big["slots"], big["do"], big["dc"], big["out"], hc=True)
        n4 = 4 * n
        so, sl = _uniform(n4, size, size)
        do, dc = _uniform(n4, size + 8, size + 8)
        raw4 = _dev(_blocks("E0", n4, size).reshape(-1))
        pk4 = torch.zeros(n4 * (size + 8), dtype=torch.uint8, device="cuda")
        out4 = torch.zeros(n4, dtype=torch.int32, device="cuda")
        off4 = torch.zeros(n4 + 1, dtype=torch.int64, device="cuda")
        batch.wrap(ctx, raw4, so, sl, pk4, do, dc, out4)
        batch.compact(ctx, pk4, do, out4, None, off4)
        ctx.set_option("hc_concurrency", 4096)
        torch.cuda.synchronize()
        assert int(off4[n4]) == n4 * (size + 8)                          # E0: every packet stored

        for _ in range(2):
            for t in (th, tw):
                for k in ("slots", "pk", "packed", "out", "off"):
                    if k in t:
                        t[k].fill_(GUARD) if t[k].dtype == torch.uint8 else t[k].zero_()
            gh.replay(); gw.replay()
            torch.cuda.synchronize()
            slots, slot = th["slots"].cpu().numpy(), oracle.bound(hc_size)
            assert [slots[i * slot:i * slot + len(w)].tobytes() for i, w in enumerate(want_hc)] == want_hc
            assert torch.equal(tw["packed"][:int(tw["off"][n])], want_pk)
        del gh, gw
    finally:
        torch.cuda.synchronize()
        ctx.close()


# ---- 6. and 7. refusals ----------------------------------------------------------------------------------------------
def test_capture_without_reserve_is_refused_and_the_capture_survives():
    from lz4net_b200 import batch, native
    torch = _torch()
    n, size = 32, 4096
    slot, td = _decode_tensors(n, size)
    _load(td, _decode_feeds(n, size, slot)[2])
    td["off"] = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    te = _encode_tensors(n, size)
    raws = _blocks("E50", n, size)
    te["raw"].copy_(_dev(raws.reshape(-1)))
    ctx = _ctx()
    try:
        launches = ctx.launches
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for refused in (lambda: batch.decode_packed(ctx, td["comp"], td["so"], td["sl"], td["dst"], td["off"], td["out"]),
                            lambda: batch.encode(ctx, te["raw"], te["so"], te["sl"], te["slots"], te["do"], te["dc"], te["out"], hc=True),
                            lambda: batch.compact(ctx, te["slots"], te["do"], te["out"], None, td["off"])):
                with pytest.raises(native.Lz4B200Error, match=r"status -1: .*lz4b200_reserve"):
                    refused()
            assert ctx.launches == launches                              # nothing enqueued
            batch.encode(ctx, te["raw"], te["so"], te["sl"], te["slots"], te["do"], te["dc"], te["out"])
        te["out"].zero_()
        g.replay()
        torch.cuda.synchronize()
        want = [oracle.encode(b.tobytes())[1] for b in raws]
        slots = te["slots"].cpu().numpy()
        assert te["out"].tolist() == [len(w) for w in want]
        assert [slots[i * slot:i * slot + len(w)].tobytes() for i, w in enumerate(want)] == want
        del g
    finally:
        torch.cuda.synchronize()
        ctx.close()


def test_synchronous_calls_refuse_a_capturing_stream():
    from lz4net_b200 import batch, native
    torch = _torch()
    n, size = 8, 4096
    te = _encode_tensors(n, size)
    raws = _blocks("ETEXT", n, size)
    te["raw"].copy_(_dev(raws.reshape(-1)))
    so, sl = np.arange(n, dtype=np.int64) * size, np.full(n, size, np.int32)
    cap = np.full(n, oracle.bound(size), np.int32)
    do = np.arange(n, dtype=np.int64) * oracle.bound(size)
    host = np.zeros(n * oracle.bound(size) + n * 16, np.uint8)
    off, out = np.zeros(n + 1, np.int64), np.zeros(n, np.int32)
    ctx = _ctx()
    try:
        ctx.reserve(n)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for refused in (lambda: batch.encode_to_host(ctx, te["raw"], so, sl, host, do, cap, out),
                            lambda: batch.stream_encode_to_host(ctx, te["raw"], block_size=4096),
                            lambda: batch.wrap_to_host_packed(ctx, te["raw"], so, sl, host, off, out)):
                with pytest.raises(native.Lz4B200Error, match=r"status -1: .*capturing stream"):
                    refused()
            batch.encode(ctx, te["raw"], te["so"], te["sl"], te["slots"], te["do"], te["dc"], te["out"])
        assert not host.any() and not out.any()
        g.replay()
        torch.cuda.synchronize()
        assert te["out"].tolist() == [len(oracle.encode(b.tobytes())[1]) for b in raws]
        del g
    finally:
        torch.cuda.synchronize()
        ctx.close()


# ---- 8. a context that never captured frees what it outgrows ---------------------------------------------------------
def _used():
    torch = _torch()
    torch.cuda.synchronize()
    free, total = torch.cuda.mem_get_info()
    return total - free


def _grown(ctx, n):
    before = _used()
    ctx.reserve(n, hc=True)
    return _used() - before


def test_scratch_growth_frees_unless_a_graph_holds_it():
    """HC arenas of n and 4n blocks (tens of MiB apart, well above the driver's allocation granularity): a context that
    never captured holds only the larger one after growing; one that captured an HC encode keeps both."""
    from lz4net_b200 import batch
    torch = _torch()
    n, size, slack = 128, 4096, 16 << 20
    sizes = {}
    for k in (n, 4 * n):
        c = _ctx()
        try:
            sizes[k] = _grown(c, k)
        finally:
            c.close()
    assert sizes[n] > 2 * slack and sizes[4 * n] > sizes[n] + 2 * slack, sizes

    never = _ctx()
    try:
        before = _used()
        never.reserve(n, hc=True)
        torch.cuda.synchronize()
        never.reserve(4 * n, hc=True)
        assert _used() - before <= sizes[4 * n] + slack, (_used() - before, sizes)
    finally:
        never.close()

    held = _ctx()
    try:
        before = _used()
        held.reserve(n, hc=True)
        t = _encode_tensors(n, size)
        g = _capture(held, lambda ctx, t: batch.encode(ctx, t["raw"], t["so"], t["sl"], t["slots"], t["do"], t["dc"], t["out"], hc=True), t)
        held.reserve(4 * n, hc=True)
        assert _used() - before >= sizes[n] + sizes[4 * n] - slack, (_used() - before, sizes)
        g.replay()
        torch.cuda.synchronize()
        assert t["out"].tolist() == [len(oracle.encode_hc(bytes(size))[1])] * n
        del g
    finally:
        torch.cuda.synchronize()
        held.close()
