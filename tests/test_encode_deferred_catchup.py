"""The fast encoder's backward catch-up (original/lz4.c:432 / :657), which runs in EMIT for 32 parked sequences at once,
one lane per sequence, and finishes long catch-ups with the whole warp.  CPU warp emulator against the oracle.

The blocks are built so that the catch-ups have known lengths.  In incompressible data the reference's find-match loop
probes with a growing step, so the positions between two probes are never inserted into the table.  Copying the bytes
in front of an inserted probe position x to the bytes in front of a later probe position y gives a match found at y
whose catch-up is exactly as long as the copy (or is stopped by the anchor, or by ref reaching position 0).  A small
model of the reference's greedy parse (checked against the oracle's bytes) confirms every planted catch-up."""
import numpy as np
import pytest

import oracle
from tests import cases, emu

LIMIT64K = 65547


def _parse(d: bytes):
    """The reference's greedy parse (LZ4_compress64kCtx / LZ4_compressCtx, no output limit).  Returns the sequences as
    (anchor, ip found, ip caught up, ref caught up, match end) and the probed positions, in order."""
    n = len(d)
    general = n >= LIMIT64K
    shift = 20 if general else 19
    table = [0] * (1 << (32 - shift))
    mv = memoryview(d)

    def word(p):
        return int.from_bytes(mv[p:p + 4], "little")

    def h(p):
        return ((word(p) * 2654435761) & 0xFFFFFFFF) >> shift

    def hit(ref, ip):
        return (not general or ref > ip - 65536) and word(ref) == word(ip)

    seqs, probes = [], []
    if n < 13:
        return seqs, probes, 0
    mflimit, matchlimit = n - 12, n - 5
    anchor = 0
    table[h(0)] = 0
    ip = 1
    while True:
        attempts, fwd = 67, ip
        while True:
            ip = fwd
            step = attempts >> 6
            attempts += 1
            fwd = ip + step
            if fwd > mflimit:
                return seqs, probes, anchor
            k = h(ip); ref = table[k]; table[k] = ip
            probes.append(ip)
            if hit(ref, ip):
                break
        found = ip
        while ip > anchor and ref > 0 and d[ip - 1] == d[ref - 1]:
            ip -= 1; ref -= 1
        while True:
            m, r = ip + 4, ref + 4
            while m < matchlimit and d[m] == d[r]:
                m += 1; r += 1
            seqs.append((anchor, found, ip, ref, m))
            anchor = m
            if m > mflimit:
                return seqs, probes, anchor
            table[h(m - 2)] = m - 2
            k = h(m); ref = table[k]; table[k] = m
            if hit(ref, m):
                ip = found = m
                continue
            break
        ip = m + 1


def _emit(d: bytes, seqs, last_anchor):
    """LZ4 block bytes of a parse, and the output position of every sequence's token."""
    out, starts = bytearray(), []

    def length(v):
        while v >= 255:
            out.append(255); v -= 255
        out.append(v)

    for anchor, _, ip, ref, m in seqs:
        lit, ml = ip - anchor, m - ip - 4
        starts.append(len(out))
        out.append((min(lit, 15) << 4) | min(ml, 15))
        if lit >= 15:
            length(lit - 15)
        out += d[anchor:ip]
        out += (ip - ref).to_bytes(2, "little")
        if ml >= 15:
            length(ml - 15)
    lit = len(d) - last_anchor
    out.append(min(lit, 15) << 4)
    if lit >= 15:
        length(lit - 15)
    out += d[last_anchor:]
    return bytes(out), starts


def _model(d: bytes):
    seqs, probes, last = _parse(d)
    out, starts = _emit(d, seqs, last)
    assert (len(out), out) == oracle.encode(d), "the parse model disagrees with the oracle"
    return seqs, probes, starts


def _catchups(d: bytes):
    """{ip found: (catch-up length, what stopped it: 'data', 'anchor' or 'ref0')}"""
    seqs, _, _ = _model(d)
    out = {}
    for anchor, found, ip, ref, _ in seqs:
        c = found - ip
        out[found] = (c, "anchor" if ip == anchor and c else "ref0" if ref == 0 and c else "data")
    return out


def _gap_probe(probes, after, c, span):
    """Index j of the first probe past `after` whose two predecessors are far enough apart: p[j-1] + 4 < y - c - 1 and
    p[j-2] + span < y - c - 1 (x = p[j-2] is the match source, y = p[j] the probe that finds it)."""
    for j in range(2, len(probes)):
        y, x = probes[j], probes[j - 2]
        if y > after and probes[j - 1] + 4 < y - c - 1 and x + span < y - c - 1 and x - c - 1 >= 0:
            return j
    raise AssertionError("no probe gap wide enough: make the block longer")


def _plant(d: np.ndarray, x: int, y: int, c: int, tail: int = 8, ref0: bool = False):
    """Copy the c bytes in front of x and `tail` bytes from x on to y - c; the byte in front differs (catch-up c)."""
    d[y - c:y + tail] = d[x - c:x + tail].copy()
    if not ref0:
        d[y - c - 1] = d[x - c - 1] ^ 0x5A


def _noise(n, seed):
    return np.random.default_rng([seed, n]).integers(0, 256, n, dtype=np.uint8)


def build_catchups(n, cs, seed, text_tail=0):
    """A block of n noise bytes with one planted catch-up of each length in cs, in order; the last text_tail bytes are
    text (many short sequences that share the EMIT batch of the last planted one).  Returns (bytes, {y: c})."""
    for s in range(seed, seed + 40):
        d = _noise(n, s)
        if text_tail:
            d[n - text_tail:] = cases.content("ETEXT", text_tail, seed=s)
        want, after = {}, 0
        for c in cs:
            _, probes, _ = _model(d.tobytes())
            j = _gap_probe(probes, after, c, 8)
            x, y = probes[j - 2], probes[j]
            assert y + 8 < n - text_tail - 16, "block too short for these catch-ups"
            _plant(d, x, y, c)
            want[y] = c
            after = y + 64
        got = _catchups(d.tobytes())
        if all(got.get(y, (None,))[0] == c for y, c in want.items()):
            return d.tobytes(), want
    raise AssertionError("no seed gave the planted catch-ups")


def build_to_end(n, c, seed):
    """One planted catch-up whose match runs to the end of the block (5 last literals): the compressed size is then
    decided by the output-limit checks of that sequence."""
    for s in range(seed, seed + 40):
        d = _noise(n, s)
        _, probes, _ = _model(d.tobytes())
        j = _gap_probe(probes, 0, c, 8)
        x, y = probes[j - 3], probes[j]                   # (three probes back: the copy does not overlap its source)
        d = d[:probes[j + 1] + 13].copy()                 # the probe at y still fits before mflimit
        _plant(d, x, y, c, tail=len(d) - y)
        if _catchups(d.tobytes()).get(y, (None,))[0] == c:
            return d.tobytes(), y
    raise AssertionError("no seed gave the planted catch-up")


def build_ref0(n, c, seed):
    """A catch-up that runs back to position 0 of the source (stopped by ref reaching 0, not by the data)."""
    for s in range(seed, seed + 40):
        d = _noise(n, s)
        _, probes, _ = _model(d.tobytes())
        x = c                                              # positions 1..66 are all probed (step 1) in noise
        if x not in probes[:66]:
            continue
        j = _gap_probe(probes, 2 * c + 80, c, 8)
        y = probes[j]
        _plant(d, x, y, c, ref0=True)
        got = _catchups(d.tobytes())
        if got.get(y) == (c, "ref0" if c else "data"):
            return d.tobytes(), y
    raise AssertionError("no seed gave the planted catch-up")


def build_anchor(n, c, seed):
    """A catch-up over the whole literal run: a match (source in the first bytes, all inserted) ends at A, then the
    bytes from A on copy the c bytes in front of a probed position x, and the byte in front of A equals the one in
    front of x - c, so only the anchor stops the catch-up."""
    z0, m, k0 = 6, 24, 4                                   # p (a probe) lands k0 bytes into the match copied from z0
    for s in range(seed, seed + 60):
        d = _noise(n, s)
        _, probes, _ = _model(d.tobytes())
        # x - c - 1 and x - c lie past the word of the probe before x; x + 8 and the word of the probe before p lie in
        # front of the first match
        j = next(j for j in range(3, len(probes)) if probes[j] > 200 and probes[j - 2] - probes[j - 3] > c + 4
                 and probes[j - 1] + 4 < probes[j] - k0 - 1 and probes[j - 2] + 8 < probes[j] - k0 - 1)
        p, x = probes[j], probes[j - 2]
        A = p - k0 + m
        if A + c + 8 >= n - 16:
            continue
        d[x - c] = d[z0 + m] ^ 1                           # the first match stops at A ...
        d[x - c - 1] = d[z0 + m - 1]                       # ... where the catch-up would go on without the anchor
        d[p - k0:A] = d[z0:z0 + m].copy()
        d[p - k0 - 1] = d[z0 - 1] ^ 0x5A
        d[A:A + c + 8] = d[x - c:x + 8].copy()
        got = _catchups(d.tobytes())
        if got.get(A + c) == (c, "anchor"):
            return d.tobytes(), A + c
    raise AssertionError("no seed gave the planted catch-up")


def _check(blocks, caps=None, **kw):
    res, outs = emu.encode(blocks, caps, **kw)
    for i, b in enumerate(blocks):
        cap = None if caps is None else caps[i]
        assert (res[i], outs[i]) == oracle.encode(b, cap=cap), (i, len(b), cap)


@pytest.fixture(scope="module")
def planted():
    """(bytes, {y: catch-up}) per block: 64 K variant and general variant (> 65 547 bytes)."""
    out = [build_catchups(20000, [0, 1, 3, 4, 5], seed=1, text_tail=3000)]
    out += [build_catchups(65536, [c], seed=10 + c, text_tail=6000) for c in (31, 32, 33)]
    out += [build_catchups(70000, [0, 1, 3, 4, 5], seed=2, text_tail=3000)]
    out += [build_catchups(240000, [64], seed=3, text_tail=4000)]
    out += [build_catchups(1600000, [210], seed=4, text_tail=4000)]
    return out


def test_planted_catchups_match_the_oracle(planted):
    blocks = [b for b, _ in planted]
    assert sorted(c for _, w in planted for c in w.values()) == [0, 0, 1, 1, 3, 3, 4, 4, 5, 5, 31, 32, 33, 64, 210]
    assert any(len(b) >= LIMIT64K for b in blocks) and any(len(b) < LIMIT64K for b in blocks)
    _check(blocks, sched_seed=5)


def test_long_and_zero_catchups_share_an_emit_batch(planted):
    """The long ones are followed by text: the same 32-sequence batch holds the long catch-up and many short or zero
    ones (and the first block holds a zero and several short ones next to each other)."""
    for b, want in planted:
        seqs, _, _ = _model(b)
        found = [s[1] for s in seqs]
        for y in want:
            k = found.index(y)
            batch = seqs[k // 32 * 32:k // 32 * 32 + 32]
            assert any(s[1] == s[2] for s in batch if s[1] != y), "no zero catch-up next to the planted one"
    for sched in (1, 2, 9):
        _check([b for b, _ in planted], sched_seed=sched)


@pytest.mark.parametrize("c", [1, 4, 5, 20, 33])
def test_catchup_stopped_by_ref_reaching_zero(c):
    b, _ = build_ref0(65536 if c > 10 else 16000, c, seed=c)
    g, _ = build_ref0(70000, c, seed=100 + c)
    _check([b, g], sched_seed=3)


@pytest.mark.parametrize("c", [1, 3, 20])
def test_catchup_stopped_by_the_anchor(c):
    b, _ = build_anchor(65536 if c > 10 else 20000, c, seed=c)
    g, _ = build_anchor(70000, c, seed=50 + c)
    _check([b, g], sched_seed=4)


def test_output_limit_around_caught_up_sequences(planted):
    """The :663 check uses the caught-up literal length: sweep the capacity byte by byte over the output of every
    planted sequence with a non-zero catch-up (general variant: the longest of its block, to keep the run short)."""
    for b, want in planted[:1] + planted[4:5]:
        seqs, _, starts = _model(b)
        found = [s[1] for s in seqs]
        caps = []
        for y, c in want.items():
            if c == 0 or (len(b) >= LIMIT64K and c != max(want.values())):
                continue
            k = found.index(y)
            lit = seqs[k][2] - seqs[k][0]                  # caught up; the literal run before it would be c longer
            caps += list(range(starts[k] + lit - 4, starts[k] + lit + lit // 255 + c + 24))
        caps = sorted(set(caps))
        _check([b] * len(caps), caps, sched_seed=8)
    # the planted sequence is the last one: every capacity around the compressed size
    for n, c in ((16000, 5), (65536, 9), (65536, 33), (70000, 6), (240000, 64)):
        b, _ = build_to_end(n, c, seed=c)
        r, _ = oracle.encode(b)
        caps = list(range(r - 12, r + 4))
        _check([b] * len(caps), caps, sched_seed=8)


@pytest.mark.parametrize("skew", [1, 2, 3, 6])
def test_catchups_unaligned_buffers(planted, skew):
    blocks = [b for b, _ in planted[:5]] + [build_ref0(16000, 7, seed=skew)[0]]
    res, outs = emu.encode(blocks, sched_seed=skew, src_skew=skew, dst_skew=16 - skew)
    for b, r, o in zip(blocks, res, outs):
        assert (r, o) == oracle.encode(b)


@pytest.mark.parametrize("tune", [(0, 0, 0), (64, 1000, 1000), (12, 1000, 0)])
def test_catchups_under_every_heuristic(planted, tune):
    """probe_max and wide_min see the literal length before the catch-up; they still only choose between equivalent
    paths."""
    _check([b for b, _ in planted[:5]] + [cases.content(m, 30000, seed=5).tobytes() for m in ("E50", "ETEXT")],
           sched_seed=6, tune=tune)


def test_catchup_never_reads_before_the_input():
    """The page in front of the block is PROT_NONE and the catch-ups run back to position 0 of the block (ref reaching
    0), at every alignment of the block's start: the backward word reads never touch a word in front of it."""
    blocks = [build_ref0(16000, c, seed=200 + c)[0] for c in (1, 2, 3, 4, 5, 9)] + [build_ref0(70000, 6, seed=7)[0]]
    for b in blocks:
        for pad in range(4):
            res, outs = emu.encode([b], sched_seed=3, fence="front", pad=pad)
            assert (res[0], outs[0]) == oracle.encode(b), (len(b), pad)
