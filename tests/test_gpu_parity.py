"""GPU parity tests (H100): every check calls liblz4b200.so through its C ABI and compares with the oracle.

Same shape as lz4net's ConformanceTests (src/LZ4.Tests/ConformanceTests.cs:57-148: all encoders byte-identical, all
decoders round-trip), WrapTests.cs:11-48, StreamTests.cs:22-63 and the upstream fuzzer's +-1 invariants
(original/fuzzer.c:176-227), with the synthetic content models of tests/cases.py instead of the Silesia corpus."""
import hashlib
import json
import os

import numpy as np
import pytest

import oracle
from tests import cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import lz4net_b200
    return lz4net_b200.default_context()


@pytest.fixture(params=[-1, 0, 1, 2], ids=["hc-auto", "hc-thread", "hc-warp-smem", "hc-warp-l1"])
def hck(ctx, request):
    """Every HC kernel of the library (lz4hc_encode.cuh: a thread per block; lz4hc_warp.cuh: a warp per block on a static
    index, block staged in shared memory / read through L1) emits the reference's bytes, and so does the default, which
    chooses per batch."""
    prev = ctx.get_option("hc_kernel")
    ctx.set_option("hc_kernel", request.param)
    yield request.param
    ctx.set_option("hc_kernel", prev)


def _inputs(models=cases.MODELS, lens=None, seed0=0):
    lens = lens or ([65536] + cases.random_lengths(6, 65546, seed=77) + [65546, 13, 12, 1, 0, 300])
    out = []
    for i, m in enumerate(models):
        for j, n in enumerate(lens):
            out.append(cases.content(m, n, seed=seed0 + 31 * i + j).tobytes())
    return out


def test_library_loaded_and_device_present():
    from lz4net_b200 import native
    assert native.lib().lz4b200_device_count() >= 1


def test_encode_fast_byte_identical(ctx):
    blocks = _inputs()
    res, outs = ctx.encode_blocks(blocks)
    for b, r, o in zip(blocks, res, outs):
        assert (r, o) == oracle.encode(b), len(b)


@pytest.mark.parametrize("variant,warps", [(1, 5), (2, 0), (1, 0), (2, 3)])
def test_encode_fast_kernel_variants(ctx, variant, warps):
    """Every form of the round (always-exact votes / resolved through the table) emits the same bytes: lz4net's.  Also with
    fewer encoder warps per SM and the prefetch off."""
    blocks = _inputs(lens=[65536, 65546, 4097, 13, 70000])
    ctx.set_option("encode_variant", variant)
    ctx.set_option("encode_ctas_per_sm", warps)
    ctx.set_option("encode_prefetch", 0 if warps == 3 else 512)
    try:
        res, outs = ctx.encode_blocks(blocks)
    finally:
        ctx.set_option("encode_variant", 2); ctx.set_option("encode_ctas_per_sm", 0); ctx.set_option("encode_prefetch", 512)
    for b, r, o in zip(blocks, res, outs):
        assert (r, o) == oracle.encode(b), (variant, warps, len(b))


def test_encode_output_limit_inside_every_emission_batch(ctx):
    """The encoder checks the reference's output limits for 32 parked sequences at a time: sweep the capacity across a
    whole block so that the first failing sequence falls at every position of such a batch."""
    d = cases.content("ETEXT", 3000, seed=5).tobytes()
    r, _ = oracle.encode(d)
    caps = list(range(0, r + 3))
    res, outs = ctx.encode_blocks([d] * len(caps), caps=caps)
    for cap, rr, o in zip(caps, res, outs):
        assert (rr, o) == oracle.encode(d, cap=cap), cap


def test_encode_hc_byte_identical(ctx, hck):
    blocks = _inputs(lens=[65536, 40000, 65546, 20, 12, 0, 100000])
    res, outs = ctx.encode_blocks(blocks, hc=True)
    for b, r, o in zip(blocks, res, outs):
        assert (r, o) == oracle.encode_hc(b), len(b)


def test_encode_general_variant_above_64k(ctx):
    blocks = [cases.content(m, n, seed=7).tobytes()
              for m, n in (("ETEXT", 65547), ("lowent", 70001), ("E50", 150000), ("periodic", 1 << 20), ("mixed", 69999),
                           ("E100", 200000), ("runs", 131072), ("E0", 66000), ("ETEXT", 1 << 20))]
    res, outs = ctx.encode_blocks(blocks)
    for b, r, o in zip(blocks, res, outs):
        assert (r, o) == oracle.encode(b), len(b)


@pytest.mark.parametrize("hc", [False, True])
def test_encode_limited_output(ctx, hc):
    """cap = exact / one short / n (LZ4Stream.cs:243-246, LZ4Codec.cs:518-523) / tiny -- same verdict and bytes."""
    fn = oracle.encode_hc if hc else oracle.encode
    blocks, caps = [], []
    for i, m in enumerate(cases.MODELS):
        for n in (200, 3000, 65536):
            d = cases.content(m, n, seed=40 + i).tobytes()
            r = fn(d)[0]
            for cap in (r, r - 1, n, n - 1, r // 2, 0, 1, 7, 8, 13):
                if cap >= 0:
                    blocks.append(d); caps.append(cap)
    res, outs = ctx.encode_blocks(blocks, caps=caps, hc=hc)
    for b, c, r, o in zip(blocks, caps, res, outs):
        assert (r, o) == fn(b, cap=c), (len(b), c)


def test_golden_vectors(ctx):
    g = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "golden_v1.json")))
    datas = [cases.AUTOTEST if c["model"] == "autotest" else cases.content(c["model"], c["n"], c["seed"]).tobytes() for c in g["cases"]]
    for mode, hc in (("fast", False), ("hc", True)):
        res, outs = ctx.encode_blocks(datas, hc=hc)
        res2, _ = ctx.encode_blocks(datas, caps=[len(d) for d in datas], hc=hc)
        for c, r, o, r2 in zip(g["cases"], res, outs, res2):
            assert r == c[mode]["len"] and hashlib.sha256(o).hexdigest() == c[mode]["sha256"], (c["name"], mode)
            assert r2 == c[mode]["len_cap_n"], (c["name"], mode)


@pytest.mark.parametrize("lanes", [32, 16, 8, 4, 132, 116, 108, 104, 1])
@pytest.mark.parametrize("known", [True, False])
def test_decode_bit_exact(ctx, lanes, known):
    ctx.set_option("decode_lanes", lanes)
    raws = _inputs(lens=[65536, 1, 12, 13, 700, 33000, 200000])
    comp = []
    for i, d in enumerate(raws):
        comp.append((oracle.encode_hc if i % 3 == 0 else oracle.encode)(d)[1])
    res, outs = ctx.decode_blocks(comp, [len(d) for d in raws], known=known)
    ctx.set_option("decode_lanes", 16)
    for c, d, r, o in zip(comp, raws, res, outs):
        assert r == (len(c) if known else len(d)), (len(d), r)
        assert o == d


def test_decode_size_invariants(ctx):
    """original/fuzzer.c:176-210: exact size works, size +-1 must fail; verdicts equal the oracle's."""
    from lz4net_b200 import synth
    for known in (True, False):
        comp, caps, expect = [], [], []
        for seed in range(8):
            d = synth.fuz_block(seed, 8000).tobytes()
            c = oracle.encode(d)[1]
            n = len(d)
            if known:
                for osz in (n, n - 1, n + 1):
                    comp.append(c); caps.append(osz); expect.append(oracle.decode_known(c, osz)[0])
            else:
                for cc, osz in ((c, n + 1), (c, n), (c, n - 1), (c[:-1], n), (c + b"\0", n)):
                    comp.append(cc); caps.append(osz); expect.append(oracle.decode_unknown(cc, osz)[0])
        res, _ = ctx.decode_blocks(comp, caps, known=known)
        for r, e in zip(res, expect):
            assert (r < 0) == (e < 0) and (e < 0 or r == e), (r, e)
        assert any(e < 0 for e in expect) and any(e >= 0 for e in expect)


@pytest.mark.parametrize("lanes", [16, 1])
@pytest.mark.parametrize("known", [True, False])
def test_decode_corrupt_streams(ctx, known, lanes):
    ctx.set_option("decode_lanes", lanes)
    rng = np.random.default_rng(5)
    comp, caps = [], []
    for i in range(400):
        d = cases.content("mixed", 2500, seed=i).tobytes()
        c = bytearray(oracle.encode(d)[1])
        kind = i % 3
        if kind == 0:
            for _ in range(int(rng.integers(1, 4))):
                c[int(rng.integers(0, len(c)))] ^= 1 << int(rng.integers(0, 8))
        elif kind == 1:
            c = c[: int(rng.integers(1, len(c)))]
        else:
            c[int(rng.integers(0, len(c)))] = 0xFF
        comp.append(bytes(c)); caps.append(len(d))
    res, outs = ctx.decode_blocks(comp, caps, known=known)
    ctx.set_option("decode_lanes_auto", 1)
    for c, cap, r, o in zip(comp, caps, res, outs):
        er, eo = (oracle.decode_known if known else oracle.decode_unknown)(c, cap)
        assert (r < 0) == (er < 0), (r, er)
        if er >= 0:
            assert r == er and o[:len(eo)] == eo


def test_decode_length_overflow_input(ctx):
    """original/fuzzer.c:96-116 (issue 52): 0x0F 00 00 then 0xFF... must be rejected, not overflow."""
    bad = bytes([0x0F, 0, 0]) + b"\xff" * (1 << 20)
    res, _ = ctx.decode_blocks([bad], [1 << 20], known=True)
    assert res[0] < 0
    res, _ = ctx.decode_blocks([bad], [1 << 20], known=False)
    assert res[0] < 0


def test_synth_device_equals_numpy(ctx):
    import torch
    from lz4net_b200 import batch, synth
    for cid, cls in enumerate(synth.CLASSES):
        for bs, nb, first in ((65536, 5, 0), (1000, 7, 123456), (65536 + 13, 3, 9)):
            t = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
            batch.synth_fill(ctx, t, nb, bs, cid, seed=42, first_block=first)
            torch.cuda.synchronize()
            want = synth.make_blocks(cls, nb, bs, seed=42, first_block=first)
            assert np.array_equal(t.cpu().numpy().reshape(nb, bs), want), (cls, bs)


@pytest.mark.parametrize("cls", ["E0", "E50", "E100", "ETEXT"])
def test_device_batch_roundtrip_and_sampled_parity(ctx, cls):
    """BASELINE config 2 shape at a size that runs in seconds: device-resident batch, encode -> compact -> decode,
    whole-batch equality on the device, byte parity with the oracle on a sample of blocks."""
    import torch
    from lz4net_b200 import batch, synth
    nb, bs = 4096, 65536
    slot = oracle.bound(bs)
    raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    batch.synth_fill(ctx, raw, nb, bs, synth.CLASS_ID[cls], seed=3)
    so, do, sl, dc = batch.uniform_layout(nb, bs, slot, "cuda")
    slots = torch.empty(nb * slot, dtype=torch.uint8, device="cuda")
    clen = torch.zeros(nb, dtype=torch.int32, device="cuda")
    batch.encode(ctx, raw, so, sl, slots, do, dc, clen)
    off = torch.zeros(nb + 1, dtype=torch.int64, device="cuda")
    packed = torch.empty(nb * slot, dtype=torch.uint8, device="cuda")
    batch.compact(ctx, slots, do, clen, packed, off)
    out = torch.zeros(nb * bs, dtype=torch.uint8, device="cuda")
    consumed = torch.zeros(nb, dtype=torch.int32, device="cuda")
    batch.decode(ctx, packed, off[:-1].contiguous(), clen, out, so, sl, consumed, known=True)
    torch.cuda.synchronize()
    assert torch.equal(off[1:] - off[:-1], clen.to(torch.int64))
    assert torch.equal(consumed, clen)
    assert torch.equal(out, raw)
    h_raw = raw.cpu().numpy().reshape(nb, bs); h_len = clen.cpu().numpy(); h_off = off.cpu().numpy(); h_packed = packed.cpu().numpy()
    for i in list(range(0, nb, 257)) + [nb - 1]:
        r, o = oracle.encode(h_raw[i])
        assert h_len[i] == r and h_packed[h_off[i]:h_off[i] + r].tobytes() == o, i


def test_encode_hc_limited_output_every_kernel(ctx, hck):
    blocks, caps = [], []
    for i, m in enumerate(("ETEXT", "lowent", "E50", "periodic", "runs", "E0")):
        d = cases.content(m, 5000, seed=40 + i).tobytes()
        r = oracle.encode_hc(d)[0]
        for cap in (r, r - 1, len(d), len(d) - 1, r // 2, 0, 1, 7, 8, 13):
            blocks.append(d); caps.append(cap)
    d = cases.content("ETEXT", 1200, seed=5).tobytes()
    for cap in range(0, oracle.encode_hc(d)[0] + 3):
        blocks.append(d); caps.append(cap)
    res, outs = ctx.encode_blocks(blocks, caps=caps, hc=True)
    for b, c, r, o in zip(blocks, caps, res, outs):
        assert (r, o) == oracle.encode_hc(b, cap=c), (len(b), c)


def test_encode_hc_handed_back_blocks(ctx, hck):
    """A run of period 3 two of whose strings share a hash bucket (the warp kernels hand such a block to the thread kernel,
    tests/test_kernels_emu.py) between ordinary blocks and blocks above 64 KiB: one batch, the reference's bytes."""
    rng = np.random.default_rng(3)
    odd = rng.integers(0, 256, 500, dtype=np.uint8).tobytes() + bytes([1, 65, 170]) * 200 + rng.integers(0, 256, 500, dtype=np.uint8).tobytes()
    blocks = []
    for i in range(40):
        blocks.append(cases.content(cases.MODELS[i % len(cases.MODELS)], 65536 if i % 3 else 3000 + i, seed=900 + i).tobytes())
        if i % 7 == 0: blocks.append(odd)
        if i % 11 == 0: blocks.append(cases.content("ETEXT", 70000 + i, seed=i).tobytes())
    res, outs = ctx.encode_blocks(blocks, hc=True)
    for b, r, o in zip(blocks, res, outs):
        assert (r, o) == oracle.encode_hc(b), len(b)


def test_device_batch_hc_sampled_parity(ctx, hck):
    import torch
    from lz4net_b200 import batch, synth
    nb, bs = 1024, 65536
    slot = oracle.bound(bs)
    raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    q = nb // 4
    for cid in range(4):
        batch.synth_fill(ctx, raw[cid * q * bs:], q, bs, cid, seed=5, first_block=cid * q)
    so, do, sl, dc = batch.uniform_layout(nb, bs, slot, "cuda")
    slots = torch.empty(nb * slot, dtype=torch.uint8, device="cuda")
    clen = torch.zeros(nb, dtype=torch.int32, device="cuda")
    batch.encode(ctx, raw, so, sl, slots, do, dc, clen, hc=True)
    out = torch.zeros(nb * bs, dtype=torch.uint8, device="cuda")
    consumed = torch.zeros(nb, dtype=torch.int32, device="cuda")
    batch.decode(ctx, slots, do, clen, out, so, sl, consumed, known=True)
    torch.cuda.synchronize()
    assert torch.equal(out, raw) and torch.equal(consumed, clen)
    h_raw = raw.cpu().numpy().reshape(nb, bs); h_len = clen.cpu().numpy(); h_slots = slots.cpu().numpy().reshape(nb, slot)
    for i in range(0, nb, 61):
        r, o = oracle.encode_hc(h_raw[i])
        assert h_len[i] == r and h_slots[i, :r].tobytes() == o, i


@pytest.mark.parametrize("cid,name", [(1, "E50"), (3, "ETEXT")])
def test_hc_kernel_chosen_on_the_device(ctx, cid, name):
    """Batches of more than three blocks per SM: a sample of the batch is looked at on the device (block sizes, hash-bucket
    depth), the thread kernel and the warp kernel are both enqueued and one of them runs; whichever does, the bytes are the
    reference's."""
    import torch
    from lz4net_b200 import batch
    assert ctx.get_option("hc_kernel") == -1
    nb, bs = 600, 65536
    slot = oracle.bound(bs)
    raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    batch.synth_fill(ctx, raw, nb, bs, cid, seed=9, first_block=0)
    so, do, sl, dc = batch.uniform_layout(nb, bs, slot, "cuda")
    slots = torch.empty(nb * slot, dtype=torch.uint8, device="cuda")
    clen = torch.zeros(nb, dtype=torch.int32, device="cuda")
    batch.encode(ctx, raw, so, sl, slots, do, dc, clen, hc=True)
    torch.cuda.synchronize()
    h_raw = raw.cpu().numpy().reshape(nb, bs); h_len = clen.cpu().numpy(); h_slots = slots.cpu().numpy().reshape(nb, slot)
    for i in list(range(0, nb, 37)) + [nb - 1]:
        r, o = oracle.encode_hc(h_raw[i])
        assert h_len[i] == r and h_slots[i, :r].tobytes() == o, (name, i)


def test_hc_large_batch_of_blocks_above_64k(ctx):
    """The same choice with a batch made of blocks the warp kernel cannot take (128 KiB): thread kernel; and with a minority
    of them among 64 KiB blocks: warp kernel, the large blocks handed back inside the call."""
    import torch
    from lz4net_b200 import batch
    for nb, bs, lens in ((500, 131072, None), (640, 131072, 65536)):
        slot = oracle.bound(bs)
        raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
        batch.synth_fill(ctx, raw, nb * (bs // 65536), 65536, 3, seed=4, first_block=0)
        so, do, sl, dc = batch.uniform_layout(nb, bs, slot, "cuda")
        if lens is not None:                      # three of four blocks use only the first 64 KiB of their slot
            sl = sl.clone(); sl[torch.arange(nb, device="cuda") % 4 != 0] = lens
        slots = torch.empty(nb * slot, dtype=torch.uint8, device="cuda")
        clen = torch.zeros(nb, dtype=torch.int32, device="cuda")
        batch.encode(ctx, raw, so, sl, slots, do, dc, clen, hc=True)
        torch.cuda.synchronize()
        h_raw = raw.cpu().numpy().reshape(nb, bs); h_len = clen.cpu().numpy(); h_slots = slots.cpu().numpy().reshape(nb, slot); h_sl = sl.cpu().numpy()
        for i in list(range(0, nb, 41)) + [nb - 1, nb - 2]:
            r, o = oracle.encode_hc(h_raw[i, :h_sl[i]])
            assert h_len[i] == r and h_slots[i, :r].tobytes() == o, (nb, i)


def test_single_block_entry_points_and_autotest(ctx):
    """The startup self-test every lz4net service must pass (src/LZ4/LZ4Codec.cs:173-239), via the LZ4Codec mirror."""
    from lz4net_b200 import LZ4Codec
    original = bytearray(cases.AUTOTEST)
    for enc, oracle_enc in ((LZ4Codec.Encode, oracle.encode), (LZ4Codec.EncodeHC, oracle.encode_hc)):
        encoded = bytearray(LZ4Codec.MaximumOutputLength(len(original)))
        n = enc(original, 0, len(original), encoded, 0, len(encoded))
        assert (n, bytes(encoded[:n])) == oracle_enc(bytes(original))
        decoded = bytearray(len(original))
        assert LZ4Codec.Decode(encoded, 0, n, decoded, 0, len(decoded), True) == len(original) and decoded == original
        decoded = bytearray(len(original))
        assert LZ4Codec.Decode(encoded, 0, n, decoded, 0, len(decoded), False) == len(original) and decoded == original
        with pytest.raises(ValueError):
            LZ4Codec.Decode(encoded, 0, n - 1, bytearray(len(original)), 0, len(original), True)
    assert LZ4Codec.Encode(bytearray(0), 0, 0, bytearray(16), 0, 16) == 0          # C# boundary: empty input -> 0
    assert LZ4Codec.Encode(bytes(original)) == oracle.encode(bytes(original))[1]
    assert LZ4Codec.Decode(LZ4Codec.EncodeHC(bytes(original)), 0, -1, len(original)) == bytes(original)
    # incompressible input with cap = n: fast -> 0, HC -> -1 (src/LZ4ps/LZ4Codec.Safe.cs:721-723)
    rnd = bytearray(cases.content("E0", 2048, 1).tobytes())
    assert LZ4Codec.Encode(rnd, 0, 2048, bytearray(2048), 0, 2048) == 0
    assert LZ4Codec.EncodeHC(rnd, 0, 2048, bytearray(2048), 0, 2048) == -1


def test_wrap_unwrap(ctx):
    """src/LZ4.Tests/WrapTests.cs:11-48: lorem, incompressible 2 KiB (stored), one-byte inputs; fast and HC."""
    from lz4net_b200 import LZ4Codec

    def ref_wrap(d, hc):
        if not d:
            return bytes(8)
        r, o = (oracle.encode_hc if hc else oracle.encode)(d, cap=len(d))
        if r >= len(d) or r <= 0:
            return len(d).to_bytes(4, "little") * 2 + d
        return len(d).to_bytes(4, "little") + r.to_bytes(4, "little") + o

    for d in (cases.LOREM, cases.content("E0", 2048, 0).tobytes(), b"a", b"", cases.AUTOTEST, cases.content("ETEXT", 70000, 1).tobytes()):
        for hc, fn in ((False, LZ4Codec.Wrap), (True, LZ4Codec.WrapHC)):
            w = fn(d)
            assert w == ref_wrap(d, hc)
            assert LZ4Codec.Unwrap(w) == d
    with pytest.raises(ValueError):
        LZ4Codec.Unwrap(b"\x01\x02\x03")


def _wrap_batch_pinned(ctx, inputs, hc):
    """lz4b200_wrap_batch into page-locked slots 5 bytes larger than the packets' capacity, filled with guard bytes: the
    packets; nothing behind a packet in its slot is written."""
    import torch
    from lz4net_b200 import codec, native
    src, lens, so = codec._pack(inputs)
    caps = lens + 8 + 5
    do = codec._offsets(caps)
    dst = torch.full((int(caps.sum()) + 16,), 0xEE, dtype=torch.uint8).pin_memory().numpy()
    out = np.zeros(len(inputs), np.int32)
    native.check(native.lib().lz4b200_wrap_batch(ctx.handle, src.ctypes.data, so.ctypes.data, lens.ctypes.data, int(hc),
                                                 dst.ctypes.data, do.ctypes.data, caps.ctypes.data, out.ctypes.data,
                                                 len(inputs)), "wrap_batch")
    for o, r, c in zip(do, out, caps):
        assert (dst[o + r:o + c] == 0xEE).all(), "a byte behind a packet changed"
    return [dst[int(o):int(o) + int(r)].tobytes() for o, r in zip(do, out)]


@pytest.mark.parametrize("hc", [False, True])
def test_wrap_unwrap_batch(ctx, hc):
    """n packets through ONE batch (lz4b200_wrap_batch / unwrap_batch): every packet is byte for byte what the per-packet
    call and the reference rule (src/LZ4/LZ4Codec.cs:510-543: stored when compression does not shrink it) produce.  With
    the default and with 1 MiB pipeline stages (a batch over several stages), into pageable and page-locked slots."""
    from lz4net_b200 import LZ4Codec, codec
    inputs = [cases.LOREM, cases.content("E0", 2048, 0).tobytes(), b"a", b"", cases.AUTOTEST, cases.content("ETEXT", 70000, 1).tobytes()]
    inputs += [cases.content(m, n, seed=3 + i).tobytes() for i, m in enumerate(cases.MODELS) for n in (1, 100, 5000, 65536)]
    wants = []
    for d in inputs:
        r, o = (oracle.encode_hc if hc else oracle.encode)(d, cap=len(d)) if d else (0, b"")
        wants.append(bytes(8) if not d else (len(d).to_bytes(4, "little") * 2 + d if (r >= len(d) or r <= 0) else len(d).to_bytes(4, "little") + r.to_bytes(4, "little") + o))
    single = LZ4Codec.WrapHC if hc else LZ4Codec.Wrap
    for chunk_mb in (128, 1):
        ctx.set_option("host_chunk_mb", chunk_mb)
        try:
            packets = codec.wrap_batch(inputs, hc=hc)
            for d, p, want in zip(inputs, packets, wants):
                assert p == want, (chunk_mb, len(d))
            assert _wrap_batch_pinned(ctx, inputs, hc) == wants, chunk_mb
            assert packets[:6] == [single(d) for d in inputs[:6]]
            assert codec.unwrap_batch(packets) == inputs
            bad = list(packets); bad[3] = b"\x01\x02\x03"
            with pytest.raises(ValueError):
                codec.unwrap_batch(bad)
        finally:
            ctx.set_option("host_chunk_mb", 128)


def _ref_stream(data, block_size, hc):
    """The LZ4Stream wire bytes, built from the oracle (src/LZ4/LZ4Stream.cs:225-269)."""
    def varint(v):
        out = bytearray()
        while True:
            b = v & 0x7F; v >>= 7
            out.append(b | (0x80 if v else 0))
            if not v:
                return bytes(out)
    out = bytearray()
    for o in range(0, len(data), block_size):
        blk = data[o:o + block_size]
        r, c = (oracle.encode_hc if hc else oracle.encode)(blk, cap=len(blk))
        comp = 0 < r < len(blk)
        out += varint((1 if comp else 0) | (2 if hc else 0)) + varint(len(blk))
        if comp:
            out += varint(r)
        out += c if comp else blk
    return bytes(out)


def _stream_encode_pinned(ctx, data, block_size, hc):
    """lz4b200_stream_encode into page-locked memory with guard bytes behind the bound: the stream; nothing behind it is
    written."""
    import torch
    from lz4net_b200 import native
    l = native.lib()
    src = np.frombuffer(bytes(data) + b"\0", np.uint8)
    cap = int(l.lz4b200_stream_bound(len(data), block_size))
    dst = torch.full((cap + 64,), 0xEE, dtype=torch.uint8).pin_memory().numpy()
    w = l.lz4b200_stream_encode(ctx.handle, src.ctypes.data, len(data), block_size, int(hc), dst.ctypes.data, cap)
    assert w >= 0 and (dst[w:] == 0xEE).all(), w
    return dst[:w].tobytes()


@pytest.mark.parametrize("hc", [False, True])
def test_lz4stream_wire_format(ctx, hc):
    """StreamTests.cs:22-63 shape: write, read back; plus byte equality of the chunk stream with the reference format.
    With the default and with 1 MiB pipeline stages (then three times the data: a stream over several stages), into
    pageable and page-locked memory."""
    data = b"".join(cases.content(m, n, seed=9).tobytes() for m, n in
                    (("ETEXT", 200000), ("E0", 70000), ("E100", 130000), ("mixed", 65536), ("lowent", 12345)))
    for chunk_mb in (128, 1):
        ctx.set_option("host_chunk_mb", chunk_mb)
        try:
            for bs in (65536, 1 << 20, 1000, 16):
                d = (data if chunk_mb == 128 else data * 3) if bs >= 1000 else data[:3000]
                s = ctx.stream_encode(d, bs, hc)
                assert s == _ref_stream(d, bs, hc), (chunk_mb, bs)
                assert _stream_encode_pinned(ctx, d, bs, hc) == s, (chunk_mb, bs)
                assert ctx.stream_decode(s) == d
        finally:
            ctx.set_option("host_chunk_mb", 128)
    assert ctx.stream_encode(b"", 65536, hc) == b"" and ctx.stream_decode(b"") == b""
    s = ctx.stream_encode(data[:100000], 65536, hc)
    with pytest.raises((EOFError, ValueError)):
        ctx.stream_decode(s[:-1])


def test_compact_scan(ctx):
    import torch
    from lz4net_b200 import batch
    rng = np.random.default_rng(1)
    for n in (1, 7, 1024, 1025, 5000, 300000):
        lens = rng.integers(-2, 700, n).astype(np.int32)
        slot = 704
        slots = torch.randint(0, 256, (n * slot,), dtype=torch.uint8, device="cuda")
        so = torch.arange(n, dtype=torch.int64, device="cuda") * slot
        tl = torch.from_numpy(lens).cuda()
        off = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
        packed = torch.zeros(int(np.maximum(lens, 0).sum()) + 16, dtype=torch.uint8, device="cuda")
        batch.compact(ctx, slots, so, tl, packed, off)
        torch.cuda.synchronize()
        want = np.concatenate([[0], np.cumsum(np.maximum(lens, 0), dtype=np.int64)])
        assert np.array_equal(off.cpu().numpy(), want)
        hs = slots.cpu().numpy().reshape(n, slot); hp = packed.cpu().numpy()
        for i in list(range(0, n, max(1, n // 50))):
            l = max(int(lens[i]), 0)
            assert np.array_equal(hp[want[i]:want[i] + l], hs[i, :l])


@pytest.mark.parametrize("hc", [False, True])
def test_lz4stream_class_random_writes_and_reads(ctx, hc):
    """src/LZ4.Tests/StreamTests.cs:47-63,148-181: random-length writes (with occasional Flush), then read everything
    back in random-length reads, normal and InteractiveRead; the wire bytes equal the reference format chunk by chunk."""
    import io
    from lz4net_b200 import LZ4Stream, LZ4StreamFlags, LZ4StreamMode
    rng = np.random.default_rng(17)
    data = b"".join(cases.content(m, n, seed=4).tobytes() for m, n in (("ETEXT", 300000), ("E0", 100000), ("mixed", 60000), ("E100", 250000)))
    for bs in (65536, 4096):
        inner = io.BytesIO()
        flags = LZ4StreamFlags.IsolateInnerStream | (LZ4StreamFlags.HighCompression if hc else 0)
        cuts = [0]
        with LZ4Stream(inner, LZ4StreamMode.Compress, flags, bs, batchBlocks=7, context=ctx) as s:
            pos = 0
            while pos < len(data):
                k = int(min(len(data) - pos, rng.integers(1, 90000)))
                s.Write(data, pos, k); pos += k
                if rng.integers(0, 6) == 0:
                    s.Flush(); cuts.append(pos)
        cuts.append(len(data))
        wire = inner.getvalue()
        # a Flush ends the current chunk: the stream is the concatenation of independently framed segments
        assert wire == b"".join(_ref_stream(data[a:b], bs, hc) for a, b in zip(cuts, cuts[1:]))
        for interactive in (False, True):
            r = LZ4Stream(io.BytesIO(wire), LZ4StreamMode.Decompress,
                          LZ4StreamFlags.InteractiveRead if interactive else LZ4StreamFlags.Default, batchBlocks=5, context=ctx)
            back = bytearray()
            while True:
                want = int(rng.integers(1, 200000))
                got = r.Read(want)
                if not got:
                    break
                assert interactive or len(got) == want or len(back) + len(got) == len(data)
                back += got
            assert bytes(back) == data
        with pytest.raises(EOFError):
            LZ4Stream(io.BytesIO(wire[:-2]), LZ4StreamMode.Decompress, context=ctx).Read(len(data) + 1)


def test_lz4stream_interactive_read_takes_one_chunk_at_a_time(ctx):
    """InteractiveRead (src/LZ4/LZ4Stream.cs:376-401): a Read returns as soon as ONE chunk is decoded -- the inner stream
    (a socket, a pipe) is not asked for the next chunk first.  The byte cap bounds the read-ahead and the write buffer of
    the batching modes; Decode with an empty output returns 0 (LZ4Codec.Safe.cs:470)."""
    import io
    from lz4net_b200 import LZ4Codec, LZ4Stream, LZ4StreamFlags, LZ4StreamMode
    bs = 4096
    data = cases.content("ETEXT", 10 * bs, seed=9).tobytes()
    wire = _ref_stream(data, bs, False)
    ends, pos = [], 0                                                  # where each chunk of the wire ends
    while pos < len(wire):
        def varint(p):
            v = sh = 0
            while True:
                b = wire[p]; p += 1; v |= (b & 0x7F) << sh; sh += 7
                if not b & 0x80:
                    return v, p
        flags, pos = varint(pos); raw_len, pos = varint(pos)
        comp_len, pos = varint(pos) if flags & 1 else (raw_len, pos)
        pos += comp_len; ends.append(pos)
    inner = io.BytesIO(wire)
    r = LZ4Stream(inner, LZ4StreamMode.Decompress, LZ4StreamFlags.InteractiveRead, batchBlocks=256, context=ctx)
    back = bytearray()
    for k in range(len(ends)):
        got = r.Read(1 << 20)
        assert len(got) == bs and inner.tell() == ends[k]              # one chunk read, one chunk returned
        back += got
    assert r.Read(10) == b"" and bytes(back) == data
    # the byte cap: 3 blocks of read-ahead per acquire although 256 chunks are allowed
    inner = io.BytesIO(wire)
    r = LZ4Stream(inner, LZ4StreamMode.Decompress, batchBlocks=256, context=ctx, maxBufferBytes=3 * bs)
    assert len(r.Read(1)) == 1 and inner.tell() == ends[2]
    assert r.Read(len(data)) == data[1:]
    # ... and 2 blocks of write buffer: the third block's first byte pushes two chunks out
    out = io.BytesIO()
    w = LZ4Stream(out, LZ4StreamMode.Compress, LZ4StreamFlags.IsolateInnerStream, bs, batchBlocks=256, context=ctx, maxBufferBytes=2 * bs)
    w.Write(data[:2 * bs]); assert out.tell() == 0
    w.Write(data[2 * bs:2 * bs + 1]); assert out.tell() == ends[1]
    w.Write(data[2 * bs + 1:]); w.Close()
    assert out.getvalue() == wire
    assert LZ4Codec.Decode(wire, 0, 10, bytearray(0), 0, 0, True) == 0


@pytest.mark.parametrize("hc", [False, True])
def test_encode_batch_packed(ctx, hc):
    """Packed host output: same per-block bytes and return values as the slot form, laid back to back in block order;
    a block that does not fit its cap contributes nothing.  Small chunks force the multi-chunk pipeline."""
    fn = oracle.encode_hc if hc else oracle.encode
    blocks = _inputs(lens=[65536, 3000, 0, 13, 40000, 65546])
    caps = []
    for i, b in enumerate(blocks):
        r = fn(b)[0]
        caps.append([oracle.bound(len(b)), len(b), r, max(r - 1, 0)][i % 4])
    ctx.set_option("host_chunk_mb", 1)
    try:
        res, off, packed = ctx.encode_blocks_packed(blocks, caps=caps, hc=hc)
    finally:
        ctx.set_option("host_chunk_mb", 256)
    pos = 0
    for b, c, r, o in zip(blocks, caps, res, off):
        er, eo = fn(b, cap=c)
        assert r == er and o == pos, (len(b), c)
        assert packed[o:o + max(r, 0)] == eo
        pos += max(r, 0)
    assert off[-1] == pos == len(packed)


def test_hc_host_batch_many_small_chunks(ctx):
    """Regression: HC launches of different pipeline stages share one state arena and must not overlap."""
    blocks = [cases.content(m, 65536, seed=70 + i).tobytes() for i, m in enumerate(cases.MODELS * 3)]
    ctx.set_option("host_chunk_mb", 1)
    try:
        res, outs = ctx.encode_blocks(blocks, hc=True)
    finally:
        ctx.set_option("host_chunk_mb", 256)
    for b, r, o in zip(blocks, res, outs):
        assert (r, o) == oracle.encode_hc(b)


def test_host_batches_in_pinned_memory(ctx):
    """Host batches whose source and destination are page-locked (torch pinned tensors, as bench.py's E2E uses): the
    copies read and write the caller's buffers directly.  Small chunks keep several pipeline stages in flight and mix
    chunks of a few large blocks with chunks of many small ones.  Every block's result and bytes are the oracle's, and
    no byte outside what a block produced changes, including the gaps left between some output slots."""
    import torch
    blocks = _inputs(lens=[65536, 3000, 0, 13, 40000, 65546, 700, 1])
    n = len(blocks)

    def excl(lens):
        return np.concatenate([[0], np.cumsum(lens, dtype=np.int64)[:-1]]).astype(np.int64)

    def pinned(nbytes, data=b""):
        a = np.full(nbytes + 16, 0xEE, np.uint8)
        a[:len(data)] = np.frombuffer(data, np.uint8)
        return torch.from_numpy(a).pin_memory()

    def check_slots(dst, do, caps, res, want, known=False):
        h = dst.numpy(); untouched = np.ones(len(h), bool)
        for o, c, r, (er, eo) in zip(do, caps, res, want):
            assert (r < 0) == (er < 0) and (er < 0 or r == er), (c, r, er)
            if er >= 0:
                assert h[o:o + len(eo)].tobytes() == eo, (c, r)
            untouched[o:o + (c if known else max(r, 0))] = False   # a known-size decode may fill its whole slot
        assert (h[untouched] == 0xEE).all()

    lens = np.array([len(b) for b in blocks], np.int32)
    so = excl(lens)
    src = pinned(int(lens.sum()), b"".join(blocks))
    gaps = np.where(np.arange(n) % 5 == 0, 8, 0)               # every fifth slot starts 8 bytes after the previous one
    ctx.set_option("host_chunk_mb", 1)
    try:
        sizes = [oracle.encode(b)[0] for b in blocks]
        caps = np.array([[oracle.bound(len(b)), len(b), r, max(r - 1, 0)][i % 4] for i, (b, r) in enumerate(zip(blocks, sizes))], np.int32)
        want = [oracle.encode(b, cap=int(c)) for b, c in zip(blocks, caps)]
        # packed: appended in block order straight into the pinned destination
        dst = pinned(int(caps.sum()))
        out = np.zeros(n, np.int32); off = np.zeros(n + 1, np.int64)
        ctx.encode_batch_packed_ptr(src.data_ptr(), so.ctypes.data, lens.ctypes.data, caps.ctypes.data, dst.data_ptr(),
                                    int(caps.sum()), off.ctypes.data, out.ctypes.data, n)
        assert np.array_equal(off, np.concatenate([[0], np.cumsum(np.maximum(out, 0), dtype=np.int64)]))
        check_slots(dst, off[:-1], caps, out, want)
        # slots: every block's bytes at dst_off[i]
        do = excl(caps + gaps) + gaps
        dst = pinned(int(do[-1] + caps[-1]))
        ctx.encode_batch_ptr(src.data_ptr(), so.ctypes.data, lens.ctypes.data, dst.data_ptr(), do.ctypes.data, caps.ctypes.data,
                             out.ctypes.data, n, device=False)
        check_slots(dst, do, caps, out, want)
        # decode, known and unknown size: an exact capacity and one byte short
        comp = [oracle.encode(b)[1] for b in blocks]
        clen = np.array([len(c) for c in comp], np.int32)
        coff = excl(clen)
        csrc = pinned(int(clen.sum()), b"".join(comp))
        for known in (True, False):
            caps = np.array([len(b) - (i % 4 == 3 and len(b) > 0) for i, b in enumerate(blocks)], np.int32)
            want = [(oracle.decode_known if known else oracle.decode_unknown)(c, int(k)) for c, k in zip(comp, caps)]
            do = excl(caps + gaps) + gaps
            dst = pinned(int(do[-1] + caps[-1]))
            ctx.decode_batch_ptr(csrc.data_ptr(), coff.ctypes.data, clen.ctypes.data, dst.data_ptr(), do.ctypes.data,
                                 caps.ctypes.data, out.ctypes.data, n, known=known, device=False)
            check_slots(dst, do, caps, out, want, known)
            assert any(r < 0 for r in out) and any(r > 0 for r in out)
    finally:
        ctx.set_option("host_chunk_mb", 128)


@pytest.mark.parametrize("cls", ["E50", "ETEXT"])
def test_large_batch_properties(ctx, cls):
    """Size-independent properties on a batch the oracle could not finish in seconds (65 536 blocks = 4 GiB): the
    round trip is exact for every decoder group size, every stream is consumed exactly, the per-block sizes are
    identical across encoder variants, and a checksum of the compressed bytes of 64 sampled blocks equals the oracle's."""
    import torch
    from lz4net_b200 import batch, synth
    nb, bs = 65536, 65536
    slot = oracle.bound(bs)
    raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    for b0 in range(0, nb, 16384):
        batch.synth_fill(ctx, raw[b0 * bs:], 16384, bs, synth.CLASS_ID[cls], seed=9, first_block=b0)
    so, do, sl, dc = batch.uniform_layout(nb, bs, slot, "cuda")
    slots = torch.empty(nb * slot, dtype=torch.uint8, device="cuda")
    clen = torch.zeros(nb, dtype=torch.int32, device="cuda")
    batch.encode(ctx, raw, so, sl, slots, do, dc, clen)
    ctx.set_option("encode_variant", 1)
    clen1 = torch.zeros(nb, dtype=torch.int32, device="cuda")
    slots1 = torch.empty(nb * slot, dtype=torch.uint8, device="cuda")
    try:
        batch.encode(ctx, raw, so, sl, slots1, do, dc, clen1)
    finally:
        ctx.set_option("encode_variant", 2)
    torch.cuda.synchronize()
    assert int((clen <= 0).sum()) == 0 and torch.equal(clen, clen1)
    del slots1
    out = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    used = torch.zeros(nb, dtype=torch.int32, device="cuda")
    try:
        for lanes in (32, 16, 108, 104, 1, 0):                    # 0: the library's own choice (picked on the device)
            if lanes:
                ctx.set_option("decode_lanes", lanes)
            else:
                ctx.set_option("decode_lanes_auto", 1)
            out.zero_()
            batch.decode(ctx, slots, do, clen, out, so, sl, used, known=True)
            torch.cuda.synchronize()
            assert torch.equal(used, clen) and torch.equal(out, raw), lanes
    finally:
        ctx.set_option("decode_lanes_auto", 1)
    idx = list(range(0, nb, nb // 64))
    h_len = clen.cpu().numpy()
    for i in idx:
        r, o = oracle.encode(raw[i * bs:(i + 1) * bs].cpu().numpy().tobytes())
        got = slots[i * slot:i * slot + int(h_len[i])].cpu().numpy().tobytes()
        assert h_len[i] == r and hashlib.sha256(got).digest() == hashlib.sha256(o).digest(), i
