"""How the device-memory entry points are entered, on an H100.

Every device-memory call takes the context's lock, asks whether its stream is capturing, admits or grows the scratch it
takes and orders itself behind the calls that share that scratch.  This pins what a caller sees of that entry:

1. The argument checks of each entry point (encode, decode and measure with LZ4B200_MEM_DEVICE, decode_batch_packed,
   compact and the three device Wrap / Unwrap calls), one table: a null context, a negative count, each pointer set to
   NULL in turn, a negative dst_total_cap, a bad mode or mem, and zero blocks with and without null pointers.  Each case
   gives its status and error text and enqueues no kernel; the zero-block packed forms set out_off[0] = 0 on the caller's
   stream.
2. Every call that takes call scratch or the HC arena is refused under capture on a context nobody reserved for, with
   E_ARG naming lz4b200_reserve and nothing enqueued, while the capture stays valid; after lz4b200_reserve(n, hc) each is
   admitted at n blocks, and the graph's replay gives what the same calls give eagerly."""
import ctypes as C

import numpy as np
import pytest

import oracle
from lz4net_b200 import synth

pytestmark = pytest.mark.gpu

OK, E_ARG = 0, -1
GUARD = 0xA5
SENTINEL = 0x5A5A5A5A
N, SIZE = 4, 4096
NULL_ARG, BAD_ARG = "null argument", "bad argument"

# name: (function, argument order, pointer arguments -> the text of the call's refusal when that one is NULL, the
#        pointers a zero-block call does not look at, fixed arguments, the text of a null context, of n < 0,
#        the extra cases: (label, changed arguments, status, text))
ENTRIES = {
    "encode": ("lz4b200_encode_batch",
               ("ctx", "src", "src_off", "src_len", "dst", "dst_off", "dst_cap", "out_len", "n", "mode", "mem", "stream"),
               dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, dst=NULL_ARG, dst_off=NULL_ARG, dst_cap=NULL_ARG,
                    out_len=NULL_ARG),
               ("src", "src_off", "src_len", "dst", "dst_off", "dst_cap", "out_len"),
               dict(mode=0, mem=1), "null context", "negative block count",
               [("bad-mode", dict(mode=7), E_ARG, "unknown encoder mode"),
                ("bad-mode-null-context", dict(mode=7, ctx=None), E_ARG, "unknown encoder mode"),
                ("bad-mem", dict(mem=9), E_ARG, "mem must be")]),
    "encode-hc": ("lz4b200_encode_batch",
                  ("ctx", "src", "src_off", "src_len", "dst", "dst_off", "dst_cap", "out_len", "n", "mode", "mem", "stream"),
                  dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, dst=NULL_ARG, dst_off=NULL_ARG, dst_cap=NULL_ARG,
                       out_len=NULL_ARG),
                  ("src", "src_off", "src_len", "dst", "dst_off", "dst_cap", "out_len"),
                  dict(mode=1, mem=1), "null context", "negative block count",
                  [("bad-mem", dict(mem=9), E_ARG, "mem must be")]),
    "decode": ("lz4b200_decode_batch",
               ("ctx", "src", "src_off", "src_len", "dst", "dst_off", "dst_cap", "out_len", "n", "known", "mem", "stream"),
               dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, dst=NULL_ARG, dst_off=NULL_ARG, dst_cap=NULL_ARG,
                    out_len=NULL_ARG),
               ("src", "src_off", "src_len", "dst", "dst_off", "dst_cap", "out_len"),
               dict(known=1, mem=1), "null context", "negative block count",
               [("bad-mem", dict(mem=9), E_ARG, "mem must be")]),
    "measure": ("lz4b200_measure_batch",
                ("ctx", "src", "src_off", "src_len", "dst_cap", "out_len", "n", "known", "mem", "stream"),
                dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, out_len=NULL_ARG,
                     dst_cap="dst_cap may be NULL only when known_len == 0"),
                ("src", "src_off", "src_len", "out_len"),
                dict(known=1, mem=1), "null context", "negative block count",
                [("bad-mem", dict(mem=9), E_ARG, "mem must be"),
                 ("null-dst_cap-null-context", dict(dst_cap=None, ctx=None), E_ARG, "dst_cap may be NULL")]),
    "decode_batch_packed": ("lz4b200_decode_batch_packed",
                            ("ctx", "src", "src_off", "src_len", "dst", "dst_total_cap", "out_off", "out_len", "n", "stream"),
                            dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, dst=NULL_ARG, out_len=NULL_ARG,
                                 out_off=BAD_ARG),
                            ("src", "src_off", "src_len", "dst", "out_len"),
                            dict(), "null context", BAD_ARG,
                            [("negative-dst_total_cap", dict(dst_total_cap=-1), E_ARG, BAD_ARG),
                             ("zero-blocks-null-out_off", dict(n=0, out_off=None), E_ARG, BAD_ARG)]),
    "compact": ("lz4b200_compact",
                ("ctx", "src", "src_off", "src_len", "dst", "out_off", "n", "stream"),
                dict(src_off=BAD_ARG, src_len=BAD_ARG, out_off=BAD_ARG),
                ("src", "dst"),
                dict(), BAD_ARG, BAD_ARG,
                [("zero-blocks-null-src_off", dict(n=0, src_off=None), E_ARG, BAD_ARG)]),
    "wrap_batch_device": ("lz4b200_wrap_batch_device",
                          ("ctx", "src", "src_off", "src_len", "hc", "dst", "dst_off", "dst_cap", "out_len", "n", "stream"),
                          dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, dst=NULL_ARG, dst_off=NULL_ARG,
                               dst_cap=NULL_ARG, out_len=NULL_ARG),
                          ("src", "src_off", "src_len", "dst", "dst_off", "dst_cap", "out_len"),
                          dict(hc=0), "null context", "negative packet count", []),
    "wrap_batch_device-hc": ("lz4b200_wrap_batch_device",
                             ("ctx", "src", "src_off", "src_len", "hc", "dst", "dst_off", "dst_cap", "out_len", "n", "stream"),
                             dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, dst=NULL_ARG, dst_off=NULL_ARG,
                                  dst_cap=NULL_ARG, out_len=NULL_ARG),
                             ("src", "src_off", "src_len", "dst", "dst_off", "dst_cap", "out_len"),
                             dict(hc=1), "null context", "negative packet count", []),
    "unwrap_batch_device": ("lz4b200_unwrap_batch_device",
                            ("ctx", "src", "src_off", "src_len", "dst", "dst_off", "dst_cap", "out_len", "n", "stream"),
                            dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, dst=NULL_ARG, dst_off=NULL_ARG,
                                 dst_cap=NULL_ARG, out_len=NULL_ARG),
                            ("src", "src_off", "src_len", "dst", "dst_off", "dst_cap", "out_len"),
                            dict(), "null context", "negative packet count", []),
    "unwrap_batch_packed": ("lz4b200_unwrap_batch_packed",
                            ("ctx", "src", "src_off", "src_len", "dst", "dst_total_cap", "out_off", "out_len", "n", "stream"),
                            dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, dst=NULL_ARG, out_len=NULL_ARG,
                                 out_off=BAD_ARG),
                            ("src", "src_off", "src_len", "dst", "out_len"),
                            dict(), "null context", "negative packet count",
                            [("negative-dst_total_cap", dict(dst_total_cap=-1), E_ARG, BAD_ARG),
                             ("negative-count-null-out_off", dict(n=-1, out_off=None), E_ARG, "negative packet count"),
                             ("zero-blocks-null-out_off", dict(n=0, out_off=None), E_ARG, BAD_ARG)]),
}
PACKED = {"decode_batch_packed", "compact", "unwrap_batch_packed"}      # zero blocks: out_off[0] = 0 on the stream


def _cases():
    """(entry, label, changed arguments, status, text or None)"""
    for name, (_fn, _order, ptrs, zero_unread, _fixed, null_ctx, neg, extra) in ENTRIES.items():
        yield name, "null-context", dict(ctx=None), E_ARG, null_ctx
        yield name, "negative-count", dict(n=-1), E_ARG, neg
        for p, text in ptrs.items():
            yield name, f"null-{p}", {p: None}, E_ARG, text
        yield name, "zero-blocks", dict(n=0), OK, None
        yield name, "zero-blocks-null-pointers", dict(n=0, **{p: None for p in zero_unread}), OK, None
        for label, change, status, text in extra:
            yield name, label, change, status, text


CASES = list(_cases())


def _torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def live():
    """A context, and device buffers for N blocks that every entry point's arguments point into."""
    from lz4net_b200.codec import Context
    torch = _torch()
    ctx = Context(0)
    slot = oracle.bound(SIZE)
    bufs = dict(src=torch.zeros(N * slot, dtype=torch.uint8, device="cuda"),
                src_off=torch.arange(N, dtype=torch.int64, device="cuda") * slot,
                src_len=torch.zeros(N, dtype=torch.int32, device="cuda"),
                dst=torch.zeros(N * slot, dtype=torch.uint8, device="cuda"),
                dst_off=torch.arange(N, dtype=torch.int64, device="cuda") * slot,
                dst_cap=torch.full((N,), slot, dtype=torch.int32, device="cuda"),
                out_len=torch.zeros(N, dtype=torch.int32, device="cuda"),
                out_off=torch.zeros(N + 1, dtype=torch.int64, device="cuda"))
    yield ctx, bufs
    torch.cuda.synchronize()
    ctx.close()


@pytest.mark.parametrize("name,label,change,status,text", CASES, ids=[f"{c[0]}/{c[1]}" for c in CASES])
def test_argument_checks(live, name, label, change, status, text):
    from lz4net_b200 import native
    torch = _torch()
    ctx, bufs = live
    fn, order, _ptrs, _zero, fixed, *_ = ENTRIES[name]
    side = torch.cuda.Stream()
    args = dict(ctx=ctx.handle, n=N, dst_total_cap=bufs["dst"].numel(), stream=side.cuda_stream, **fixed)
    args.update({k: v.data_ptr() for k, v in bufs.items()})
    args.update(change)
    bufs["out_off"][0] = SENTINEL
    torch.cuda.synchronize()
    before = ctx.launches
    rc = getattr(native.lib(), fn)(*[args[k] for k in order])
    assert rc == status, (rc, native.last_error())
    if text is not None:
        assert text in native.last_error()
    side.synchronize()
    assert ctx.launches == before                                       # no kernel enqueued
    zero_packed = status == OK and name in PACKED
    assert int(bufs["out_off"][0]) == (0 if zero_packed else SENTINEL)  # only a zero-block packed form writes out_off[0]


# ---- refusal under capture, then admission after lz4b200_reserve ---------------------------------------------------
def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a)).cuda()


def _scratch_users(n, size):
    """Tensors, and the calls that take call scratch or the HC arena: name -> (call(ctx, t), its output tensors)."""
    from lz4net_b200 import batch
    from lz4net_b200.codec import Context, wrap_batch
    torch = _torch()
    raws = synth.make_blocks("ETEXT", n, size, seed=13)
    slot, pslot = oracle.bound(size), size + 8
    comp, clen = np.zeros(n * slot, np.uint8), np.zeros(n, np.int32)
    for i, b in enumerate(raws):
        r, o = oracle.encode(b.tobytes())
        comp[i * slot:i * slot + r], clen[i] = np.frombuffer(o, np.uint8), r
    ref = Context(0)
    try:
        pk = wrap_batch([b.tobytes() for b in raws], hc=False, ctx=ref)
    finally:
        ref.close()
    pkt, plen = np.zeros(n * pslot, np.uint8), np.zeros(n, np.int32)
    for i, p in enumerate(pk):
        pkt[i * pslot:i * pslot + len(p)], plen[i] = np.frombuffer(p, np.uint8), len(p)
    u8 = lambda k: torch.zeros(k, dtype=torch.uint8, device="cuda")               # noqa: E731
    i32 = lambda k: torch.zeros(k, dtype=torch.int32, device="cuda")              # noqa: E731
    i64 = lambda k: torch.zeros(k, dtype=torch.int64, device="cuda")              # noqa: E731
    stride = lambda s: torch.arange(n, dtype=torch.int64, device="cuda") * s      # noqa: E731
    full = lambda v: torch.full((n,), v, dtype=torch.int32, device="cuda")        # noqa: E731
    t = dict(raw=_dev(raws.reshape(-1)), rso=stride(size), rsl=full(size), comp=_dev(comp), cso=stride(slot), csl=_dev(clen),
             pk=_dev(pkt), pso=stride(pslot), psl=_dev(plen), sdo=stride(slot), sdc=full(slot), pdo=stride(pslot),
             pdc=full(pslot), rdo=stride(size), rdc=full(size),
             hc_slots=u8(n * slot), hc_out=i32(n),
             dp_dst=u8(n * size), dp_off=i64(n + 1), dp_out=i32(n),
             cp_packed=u8(n * slot), cp_off=i64(n + 1),
             wr_pk=u8(n * pslot), wr_out=i32(n),
             wh_pk=u8(n * pslot), wh_out=i32(n),
             uw_dst=u8(n * size), uw_out=i32(n),
             up_dst=u8(n * size), up_off=i64(n + 1), up_out=i32(n))
    calls = {
        "encode-hc": (lambda ctx, t: batch.encode(ctx, t["raw"], t["rso"], t["rsl"], t["hc_slots"], t["sdo"], t["sdc"], t["hc_out"],
                                                  hc=True), ("hc_slots", "hc_out")),
        "wrap_batch_device-hc": (lambda ctx, t: batch.wrap(ctx, t["raw"], t["rso"], t["rsl"], t["wh_pk"], t["pdo"], t["pdc"],
                                                           t["wh_out"], hc=True), ("wh_pk", "wh_out")),
        "decode_batch_packed": (lambda ctx, t: batch.decode_packed(ctx, t["comp"], t["cso"], t["csl"], t["dp_dst"], t["dp_off"],
                                                                   t["dp_out"]), ("dp_dst", "dp_off", "dp_out")),
        "compact": (lambda ctx, t: batch.compact(ctx, t["comp"], t["cso"], t["csl"], t["cp_packed"], t["cp_off"]),
                    ("cp_packed", "cp_off")),
        "wrap_batch_device": (lambda ctx, t: batch.wrap(ctx, t["raw"], t["rso"], t["rsl"], t["wr_pk"], t["pdo"], t["pdc"],
                                                        t["wr_out"]), ("wr_pk", "wr_out")),
        "unwrap_batch_device": (lambda ctx, t: batch.unwrap(ctx, t["pk"], t["pso"], t["psl"], t["uw_dst"], t["rdo"], t["rdc"],
                                                            t["uw_out"]), ("uw_dst", "uw_out")),
        "unwrap_batch_packed": (lambda ctx, t: batch.unwrap_packed(ctx, t["pk"], t["pso"], t["psl"], t["up_dst"], t["up_off"],
                                                                   t["up_out"]), ("up_dst", "up_off", "up_out")),
    }
    return raws, t, calls


def _guard(t, outs):
    for k in outs:
        t[k].fill_(GUARD) if t[k].dtype == _torch().uint8 else t[k].fill_(-7)


def test_every_scratch_user_is_refused_without_reserve_and_admitted_after():
    from lz4net_b200 import batch, native
    from lz4net_b200.codec import Context
    torch = _torch()
    n, size = 16, 4096
    raws, t, calls = _scratch_users(n, size)
    slot = oracle.bound(size)
    fast = dict(slots=torch.zeros(n * slot, dtype=torch.uint8, device="cuda"), out=torch.zeros(n, dtype=torch.int32, device="cuda"))
    outs = [k for _call, o in calls.values() for k in o]
    ctx = Context(0)
    try:
        # a fresh context: every scratch user is refused, enqueues nothing, and the capture goes on
        _guard(t, outs)
        torch.cuda.synchronize()
        launches = ctx.launches
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for name, (call, _o) in calls.items():
                with pytest.raises(native.Lz4B200Error, match=r"status -1: .*lz4b200_reserve"):
                    call(ctx, t)
                assert ctx.launches == launches, name
            batch.encode(ctx, t["raw"], t["rso"], t["rsl"], fast["slots"], t["sdo"], t["sdc"], fast["out"])
        g.replay()
        torch.cuda.synchronize()
        want = [oracle.encode(b.tobytes())[1] for b in raws]
        got = fast["slots"].cpu().numpy()
        assert fast["out"].tolist() == [len(w) for w in want]
        assert [got[i * slot:i * slot + len(w)].tobytes() for i, w in enumerate(want)] == want
        for k in outs:                                                   # the refused calls left nothing in the graph
            assert (t[k] == (GUARD if t[k].dtype == torch.uint8 else -7)).all(), k
        del g

        # reserved for n blocks with HC: each is admitted at n blocks, and the replay gives what eager calls give
        ctx.reserve(n, hc=True)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for call, _o in calls.values():
                call(ctx, t)
        _guard(t, outs)
        want = {k: v.clone() for k, v in t.items()}
        g.replay()
        ref = Context(0)
        try:
            for call, _o in calls.values():
                call(ref, want)
            torch.cuda.synchronize()
        finally:
            ref.close()
        for k in outs:
            assert torch.equal(t[k], want[k]), k
        assert t["dp_out"].tolist() == [size] * n and t["up_out"].tolist() == [size] * n
        assert t["dp_dst"].cpu().numpy().tobytes() == raws.tobytes()
        del g
    finally:
        torch.cuda.synchronize()
        ctx.close()
