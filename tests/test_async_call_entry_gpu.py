"""How the asynchronous calls between device memory and page-locked host memory check their arguments, on an H100.

One table for the six calls (the packed encode and the packed Wrap from device memory, the decode, the packed decode, the
Unwrap and the packed Unwrap into device memory): a null context, a negative count, each pointer set to NULL in turn, a
negative dst_total_cap, a bad mode, a negative length, a source or destination of the wrong kind of memory (pageable
memory where page-locked memory is required, device memory where host memory is, and the reverse), and zero blocks with
and without null pointers.  Each case gives its status and error text and enqueues no kernel; only the zero-block packed
forms write out_off[0] = 0, on the caller's stream."""
import numpy as np
import pytest

import oracle

pytestmark = pytest.mark.gpu

OK, E_ARG = 0, -1
SENTINEL = 0x5A5A5A5A
N, SIZE = 4, 4096
NULL_ARG, BAD_ARG = "null argument", "bad argument"
DEV_SRC = "src must be device memory of the context's GPU"
DEV_DST = "dst must be device memory of the context's GPU"
PINNED_SRC = "src must be page-locked host memory the device can address"
PINNED_DST = "dst must be page-locked host memory the device can address"
OUT_OFF = "out_off must be device memory of the context's GPU or page-locked host memory"
OUT_LEN = "out_len must be device memory of the context's GPU or page-locked host memory"
WRAP_LEN = "input length: negative, or a packet above INT32_MAX bytes"

# The buffers (see `live`): d_* device memory, p_* page-locked host memory, h_* pageable host memory; the offset, length
# and capacity arrays are host arrays, read during the call.
LANDED = dict(src="d_src", dst="p_dst", out_off="d_out_off", out_len="d_out_len")      # device memory -> page-locked
STAGED = dict(src="p_src", dst="d_dst", out_off="d_out_off", out_len="d_out_len")      # page-locked -> device memory
LANDED_KINDS = [("pageable-src", dict(src="h_src"), DEV_SRC), ("page-locked-src", dict(src="p_src"), DEV_SRC),
                ("device-dst", dict(dst="d_dst"), PINNED_DST), ("pageable-dst", dict(dst="h_dst"), PINNED_DST),
                ("pageable-out_off", dict(out_off="h_out_off"), OUT_OFF), ("pageable-out_len", dict(out_len="h_out_len"), OUT_LEN)]
STAGED_KINDS = [("pageable-src", dict(src="h_src"), PINNED_SRC), ("device-src", dict(src="d_src"), PINNED_SRC),
                ("page-locked-dst", dict(dst="p_dst"), DEV_DST), ("pageable-dst", dict(dst="h_dst"), DEV_DST),
                ("pageable-out_len", dict(out_len="h_out_len"), OUT_LEN)]
STAGED_PACKED_KINDS = STAGED_KINDS + [("pageable-out_off", dict(out_off="h_out_off"), OUT_OFF)]

# name: (function, argument order, buffers, pointer arguments -> the text of the call's refusal when that one is NULL, the
#        pointers a zero-block call does not look at, fixed arguments, the text of a null context, of n < 0, of a negative
#        length, whether a zero-block call writes out_off[0], the extra cases: (label, changed arguments, status, text))
ENTRIES = {
    "encode_packed_async": (
        "lz4b200_encode_batch_packed_from_device_async",
        ("ctx", "src", "src_off", "src_len", "dst_cap", "dst", "dst_total_cap", "out_off", "out_len", "n", "mode", "stream"),
        LANDED, dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, dst_cap=NULL_ARG, dst=NULL_ARG, out_len=NULL_ARG,
                     out_off=BAD_ARG),
        ("src", "src_off", "src_len", "dst_cap", "dst", "out_len"), dict(mode=0),
        "null context", BAD_ARG, "negative block length", True,
        [("negative-dst_total_cap", dict(dst_total_cap=-1), E_ARG, BAD_ARG),
         ("negative-dst_cap", dict(dst_cap="neg_len"), E_ARG, "negative block length"),
         ("bad-mode", dict(mode=7), E_ARG, "unknown encoder mode"),
         ("bad-mode-null-context", dict(mode=7, ctx=None), E_ARG, "null context"),
         ("bad-mode-negative-count", dict(mode=7, n=-1), E_ARG, "unknown encoder mode"),
         ("zero-blocks-null-out_off", dict(n=0, out_off=None), E_ARG, BAD_ARG)] +
        [(label, change, E_ARG, text) for label, change, text in LANDED_KINDS]),
    "encode_packed_async-hc": (
        "lz4b200_encode_batch_packed_from_device_async",
        ("ctx", "src", "src_off", "src_len", "dst_cap", "dst", "dst_total_cap", "out_off", "out_len", "n", "mode", "stream"),
        LANDED, dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, dst_cap=NULL_ARG, dst=NULL_ARG, out_len=NULL_ARG,
                     out_off=BAD_ARG),
        ("src", "src_off", "src_len", "dst_cap", "dst", "out_len"), dict(mode=1),
        "null context", BAD_ARG, "negative block length", True,
        [("negative-dst_total_cap", dict(dst_total_cap=-1), E_ARG, BAD_ARG),
         ("pageable-src", dict(src="h_src"), E_ARG, DEV_SRC)]),
    "wrap_packed_async": (
        "lz4b200_wrap_batch_packed_from_device_async",
        ("ctx", "src", "src_off", "src_len", "hc", "dst", "dst_total_cap", "out_off", "out_len", "n", "stream"),
        LANDED, dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, dst=NULL_ARG, out_len=NULL_ARG, out_off=BAD_ARG),
        ("src", "src_off", "src_len", "dst", "out_len"), dict(hc=0),
        "null context", BAD_ARG, WRAP_LEN, True,
        [("negative-dst_total_cap", dict(dst_total_cap=-1), E_ARG, BAD_ARG),
         ("packet-above-int32", dict(src_len="huge_len"), E_ARG, WRAP_LEN),
         ("zero-blocks-null-out_off", dict(n=0, out_off=None), E_ARG, BAD_ARG)] +
        [(label, change, E_ARG, text) for label, change, text in LANDED_KINDS]),
    "wrap_packed_async-hc": (
        "lz4b200_wrap_batch_packed_from_device_async",
        ("ctx", "src", "src_off", "src_len", "hc", "dst", "dst_total_cap", "out_off", "out_len", "n", "stream"),
        LANDED, dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, dst=NULL_ARG, out_len=NULL_ARG, out_off=BAD_ARG),
        ("src", "src_off", "src_len", "dst", "out_len"), dict(hc=1),
        "null context", BAD_ARG, WRAP_LEN, True,
        [("device-dst", dict(dst="d_dst"), E_ARG, PINNED_DST)]),
    "decode_async": (
        "lz4b200_decode_batch_to_device_async",
        ("ctx", "src", "src_off", "src_len", "dst", "dst_off", "dst_cap", "out_len", "n", "known", "stream"),
        STAGED, dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, dst=NULL_ARG, dst_off=NULL_ARG, dst_cap=NULL_ARG,
                     out_len=NULL_ARG),
        ("src", "src_off", "src_len", "dst", "dst_off", "dst_cap", "out_len"), dict(known=1),
        "null context", "negative block count", "negative block length", False,
        [("negative-dst_cap", dict(dst_cap="neg_len"), E_ARG, "negative block length"),
         ("unknown-size-negative-length", dict(known=0, src_len="neg_len"), E_ARG, "negative block length")] +
        [(label, change, E_ARG, text) for label, change, text in STAGED_KINDS]),
    "decode_packed_async": (
        "lz4b200_decode_batch_packed_to_device_async",
        ("ctx", "src", "src_off", "src_len", "dst", "dst_total_cap", "out_off", "out_len", "n", "stream"),
        STAGED, dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, dst=NULL_ARG, out_len=NULL_ARG, out_off=BAD_ARG),
        ("src", "src_off", "src_len", "dst", "out_len"), dict(),
        "null context", BAD_ARG, "negative block length", True,
        [("negative-dst_total_cap", dict(dst_total_cap=-1), E_ARG, BAD_ARG),
         ("zero-blocks-null-out_off", dict(n=0, out_off=None), E_ARG, BAD_ARG)] +
        [(label, change, E_ARG, text) for label, change, text in STAGED_PACKED_KINDS]),
    "unwrap_async": (
        "lz4b200_unwrap_batch_to_device_async",
        ("ctx", "src", "src_off", "src_len", "dst", "dst_off", "dst_cap", "out_len", "n", "stream"),
        STAGED, dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, dst=NULL_ARG, dst_off=NULL_ARG, dst_cap=NULL_ARG,
                     out_len=NULL_ARG),
        ("src", "src_off", "src_len", "dst", "dst_off", "dst_cap", "out_len"), dict(),
        "null context", "negative packet count", "negative packet length", False,
        [("negative-dst_cap", dict(dst_cap="neg_len"), E_ARG, "negative packet length")] +
        [(label, change, E_ARG, text) for label, change, text in STAGED_KINDS]),
    "unwrap_packed_async": (
        "lz4b200_unwrap_batch_packed_to_device_async",
        ("ctx", "src", "src_off", "src_len", "dst", "dst_total_cap", "out_off", "out_len", "n", "stream"),
        STAGED, dict(src=NULL_ARG, src_off=NULL_ARG, src_len=NULL_ARG, dst=NULL_ARG, out_len=NULL_ARG, out_off=BAD_ARG),
        ("src", "src_off", "src_len", "dst", "out_len"), dict(),
        "null context", BAD_ARG, "negative packet length", True,
        [("negative-dst_total_cap", dict(dst_total_cap=-1), E_ARG, BAD_ARG),
         ("negative-count-null-out_off", dict(n=-1, out_off=None), E_ARG, BAD_ARG),
         ("zero-blocks-null-out_off", dict(n=0, out_off=None), E_ARG, BAD_ARG)] +
        [(label, change, E_ARG, text) for label, change, text in STAGED_PACKED_KINDS]),
}


def _cases():
    """(entry, label, changed arguments, status, text or None)"""
    for name, (_fn, _order, _bufs, ptrs, zero_unread, _fixed, null_ctx, neg, neg_len, _packed, extra) in ENTRIES.items():
        yield name, "null-context", dict(ctx=None), E_ARG, null_ctx
        yield name, "negative-count", dict(n=-1), E_ARG, neg
        for p, text in ptrs.items():
            yield name, f"null-{p}", {p: None}, E_ARG, text
        yield name, "negative-length", dict(src_len="neg_len"), E_ARG, neg_len
        yield name, "zero-blocks", dict(n=0), OK, None
        yield name, "zero-blocks-null-pointers", dict(n=0, **{p: None for p in zero_unread}), OK, None
        for label, change, status, text in extra:
            yield name, label, change, status, text


CASES = list(_cases())


@pytest.fixture(scope="module")
def live():
    """A context, and buffers for N blocks of every kind of memory the six calls' arguments may point into."""
    import torch
    from lz4net_b200.codec import Context
    ctx = Context(0)
    slot = oracle.bound(SIZE) + 8
    pinned = lambda t: t.pin_memory()                                                   # noqa: E731
    bufs = dict(d_src=torch.zeros(N * slot, dtype=torch.uint8, device="cuda"),
                p_src=pinned(torch.zeros(N * slot, dtype=torch.uint8)),
                h_src=np.zeros(N * slot, np.uint8),
                d_dst=torch.zeros(N * slot, dtype=torch.uint8, device="cuda"),
                p_dst=pinned(torch.zeros(N * slot, dtype=torch.uint8)),
                h_dst=np.zeros(N * slot, np.uint8),
                d_out_off=torch.zeros(N + 1, dtype=torch.int64, device="cuda"),
                h_out_off=np.zeros(N + 1, np.int64),
                d_out_len=torch.zeros(N, dtype=torch.int32, device="cuda"),
                h_out_len=np.zeros(N, np.int32),
                src_off=np.arange(N, dtype=np.int64) * slot,
                src_len=np.full(N, SIZE, np.int32),
                dst_off=np.arange(N, dtype=np.int64) * slot,
                dst_cap=np.full(N, slot, np.int32),
                neg_len=np.array([SIZE, -1] + [SIZE] * (N - 2), np.int32),
                huge_len=np.array([SIZE, 2**31 - 8] + [SIZE] * (N - 2), np.int32))
    yield ctx, bufs
    torch.cuda.synchronize()
    ctx.close()


def _address(b):
    return b.data_ptr() if hasattr(b, "data_ptr") else b.ctypes.data


@pytest.mark.parametrize("name,label,change,status,text", CASES, ids=[f"{c[0]}/{c[1]}" for c in CASES])
def test_argument_checks(live, name, label, change, status, text):
    import torch
    from lz4net_b200 import native
    ctx, bufs = live
    fn, order, kinds, _ptrs, _zero, fixed, _nc, _neg, _nl, packed, _extra = ENTRIES[name]
    side = torch.cuda.Stream()
    named = dict(kinds, src_off="src_off", src_len="src_len", dst_off="dst_off", dst_cap="dst_cap")
    named.update({k: v for k, v in change.items() if isinstance(v, str)})
    args = dict(ctx=ctx.handle, n=N, dst_total_cap=N * (oracle.bound(SIZE) + 8), stream=side.cuda_stream, **fixed)
    args.update({k: _address(bufs[b]) for k, b in named.items()})
    args.update({k: v for k, v in change.items() if not isinstance(v, str)})
    bufs["d_out_off"][0] = SENTINEL
    torch.cuda.synchronize()
    before = ctx.launches
    rc = getattr(native.lib(), fn)(*[args[k] for k in order])
    assert rc == status, (rc, native.last_error())
    if text is not None:
        assert text in native.last_error()
    side.synchronize()
    assert ctx.launches == before                                       # no kernel enqueued
    zero_packed = status == OK and packed
    assert int(bufs["d_out_off"][0]) == (0 if zero_packed else SENTINEL)  # only a zero-block packed form writes out_off[0]
