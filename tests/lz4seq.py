"""Constructed LZ4 block streams -- TEST INFRASTRUCTURE ONLY.

Encoders never aim at the decoders' thresholds: the greedy and HC parsers stop matching 12 bytes before the end, pick
offsets and lengths the data gives them, and put sequence headers wherever the parse happens to be.  build() writes raw
sequences verbatim instead -- any literal run, any offset (0 and op + 1 included), any match length -- and corpus() uses
it to put a byte exactly on each accept / reject rule of the reference decoders (original/lz4.c:812-1044) and on each
internal threshold of the kernels (lz4_decode.cuh, lz4_decode_lpb.cuh, lz4_measure.cuh).

A case is (name, stream, cap): every decoder takes it both as a known-size decode (cap = the decoded size) and as an
unknown-size one (cap = the capacity).  The corpus is a pure function of its seed; tests/golden/constructed_v1.json
holds what the reference returned on it (tests/golden/make_golden.py).
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np

MINMATCH = 4


class Case(NamedTuple):
    name: str
    stream: bytes
    cap: int


def _length_bytes(x: int) -> bytes:
    """The 255-continuation encoding of a length beyond the token's 15."""
    return b"\xff" * (x // 255) + bytes([x % 255])


def build(sequences, last_literals=b"") -> bytes:
    """A raw LZ4 block: one sequence per (literals, offset, match_length) -- match_length counts MINMATCH, offset is
    written as its low 16 bits, unchecked -- then a final token with `last_literals`."""
    out = bytearray()
    for lits, off, mlen in sequences:
        L, M = len(lits), mlen - MINMATCH
        assert M >= 0
        out.append((min(L, 15) << 4) | min(M, 15))
        if L >= 15:
            out += _length_bytes(L - 15)
        out += lits
        out += bytes([off & 255, (off >> 8) & 255])
        if M >= 15:
            out += _length_bytes(M - 15)
    L = len(last_literals)
    out.append(min(L, 15) << 4)
    if L >= 15:
        out += _length_bytes(L - 15)
    out += last_literals
    return bytes(out)


def decoded_size(sequences, last_literals=b"") -> int:
    return sum(len(l) + m for l, _, m in sequences) + len(last_literals)


def header_size(L: int, mlen: int) -> int:
    """Stream bytes of one sequence other than its literals: token, length bytes, offset."""
    M = mlen - MINMATCH
    return 1 + (len(_length_bytes(L - 15)) if L >= 15 else 0) + 2 + (len(_length_bytes(M - 15)) if M >= 15 else 0)


class _Gen:
    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.cases = []

    def lits(self, n):
        return self.rng.integers(0, 256, n, dtype=np.uint8).tobytes()

    def prefix(self, n):
        """Sequences whose output is n >= 13 bytes, mostly fresh data: literal runs of at most 31 bytes, each with a short
        match.  (A longer run would be copied by the whole warp in the lpb decoder, which then serves every match that
        reaches behind the run from global memory instead of from its output ring.)"""
        seqs = []
        while n > 36:
            seqs.append((self.lits(20), 5, 4))
            n -= 24
        return seqs + [(self.lits(n - 5), 3, 5)]

    def add(self, name, seqs, last, caps=(0,)):
        s = build(seqs, last)
        n = decoded_size(seqs, last)
        for d in caps:
            self.cases.append(Case(f"{name}/cap{d:+d}", s, n + d))


# cap deltas around the decoded size: exact, +-1, the known-size last-literal window (8), the unknown-size one (12)
TAIL_CAPS = (-1, 0, 1, 4, 5, 7, 8, 11, 12, 13)


def _tail(g):
    """The end-of-block rules.  The last sequence (L literals, a match of M) is followed by t last literals, t = 0..13,
    under caps of n - 1 .. n + 13.  Known size: literal end at cap, cap - 8, cap - 9 with a match ending at cap - 5 or
    cap - 4.  Unknown size: literal end at cap - 11 / cap - 12, ip + L at isize - 8 / isize - 9, and match-length bytes
    (M = 19: one byte of 0; 20: one of 1; 274, 275: 255 then 0 / 1; 529: 255, 255, 0) on both sides of isize - 6."""
    for L in (0, 5):
        for mlen in (4, 19, 20, 274, 275, 529):
            for t in range(14):
                seqs = g.prefix(24 + (t & 3)) + [(g.lits(L), 1 if mlen > 8 else 7, mlen)]
                g.add(f"tail/L{L}/M{mlen}/t{t}", seqs, g.lits(t), TAIL_CAPS)
    # Decodable at an unlimited capacity, rejected at a capacity of exactly the decoded size, which the packed unknown-size
    # decode once gave each block: the last sequence's literal run ends 9 bytes before the end, within 12 bytes of the
    # capacity, so the unknown-size rules take it for the block's last run.
    g.add("tail/packed-capacity/forced-last-literals-cap-12", g.prefix(30) + [(g.lits(3), 7, 4)], g.lits(5), (0, 2, 3, 12))
    # the block is nothing but literals: cap = L is the only accepted known size; unknown size takes cap >= L
    for L in (0, 1, 5, 12, 13, 14, 15, 16, 270):
        g.add(f"tail/only-literals/L{L}", [], g.lits(L), (-1, 0, 1, 12))


def _offsets(g):
    """Match offsets.  1..8 (overlapping copies, the lpb per-word path below 8 and the carry loop above), L - 1 / L / L + 1
    (the group fast path forwards a match from the ring when off <= L), M - 1 / M / M + 1 (the copy is overlap-free
    when off >= M), op (accepted: the block's first byte), op + 1 and 0 (rejected).  far: the sequence sits where
    every fast path runs; near: it is the block's last one, on the careful / general code."""
    i = 0
    for L in (0, 1, 7, 16, 32, 33):
        for mlen in (4, 5, 8, 17, 32, 33, 64, 65):
            op = 40 + (i & 3) + L
            i += 1
            offs = set(range(1, 9)) | {L - 1, L, L + 1, mlen - 1, mlen, mlen + 1, op, op + 1, 0}
            for off in sorted(o for o in offs if 0 <= o <= op + 1):
                for where, last in (("far", 120), ("near", 5)):
                    seqs = g.prefix(op - L) + [(g.lits(L), off, mlen)]
                    g.add(f"offset/L{L}/M{mlen}/off{off}/{where}", seqs, g.lits(last))


def _ring_window(g):
    """Offsets at the lane-per-block decoder's output window: the kernel geometry serves matches up to WIN = 248 bytes
    back from its 256-byte ring, the emulator's second geometry up to 504 from 512; the ring's last words (up to 256 /
    512 back) hold bytes the write cursor's partial word has already overwritten.  The write cursor is at every byte
    phase (prefix + 0..3), the match in the fast region (far) and as the last sequence (near, where the general code
    runs)."""
    for off in (248, 249, 250, 252, 253, 254, 255, 256, 257, 504, 505, 508, 509, 510, 511, 512, 513):
        for mlen in (4, 13, 32, 33, 64):
            for r in range(4):
                for where, last in (("far", 120), ("near", 5)):
                    seqs = g.prefix(600 + r) + [(g.lits(3), off, mlen)]
                    g.add(f"ring/off{off}/M{mlen}/r{r}/{where}", seqs, g.lits(last))
    # offset 65535 inside blocks of 100-200 KiB
    for n, mlen in ((100_000, 4), (150_000, 300), (200_000, 70_000)):
        seqs = g.prefix(66_000) + [(g.lits(7), 65535, mlen), (g.lits(2), 65534, 33), (g.lits(40), 65535, 64)]
        fill = n - decoded_size(seqs)
        seqs += [(g.lits(100), 60_000 + 91 * k % 5000, 1000) for k in range(max(fill // 1100 - 1, 0))]
        g.add(f"ring/off65535/n{n}", seqs, g.lits(64), (0, 1))


def _lengths(g):
    """Literal runs and matches at the length-code boundaries: 14-16 (code 15), 31-33 and 63-65 (the fast paths' 32 / 64),
    269-271 and 15 + 255k (a continuation byte of 255 followed by 0); matches of 18 / 19 (code 15), 64 / 65, 273-275;
    long runs of 1 KiB .. 70 KiB with periods of 1-8 bytes."""
    lit_lens = (14, 15, 16, 31, 32, 33, 63, 64, 65, 269, 270, 271, 15 + 2 * 255, 15 + 3 * 255)
    for L in lit_lens:
        for mlen in (4, 18, 19, 64, 65, 273, 274, 275):
            for off in (1, 16, 40 + L):
                seqs = g.prefix(40) + [(g.lits(L), off, mlen), (g.lits(3), 9, 6)]
                g.add(f"length/L{L}/M{mlen}/off{off}", seqs, g.lits(70))
    for mlen in (1024, 4096, 70_000):
        for period in range(1, 9):
            seqs = g.prefix(20) + [(g.lits(period + 1), period, mlen), (g.lits(4), 3, 4)]
            g.add(f"length/run{mlen}/p{period}", seqs, g.lits(30), (0, 1))


def _dense(g, n_seqs):
    """Short sequences of varying shape (headers 1-3 bytes): consecutive headers fall on every phase of a boundary."""
    out = []
    for i in range(n_seqs):
        L = (0, 1, 3, 15, 2, 8)[i % 6]
        mlen = (4, 19, 7, 12, 64, 5, 20)[i % 7]
        out.append((g.lits(L), 1 + (i * 7) % 24, mlen))
    return out


def _placement(g):
    """A sequence header k = 0..8 bytes before each TMA chunk boundary of the group decoders (1024 / 512 / 256 / 128 for
    G = 32 / 16 / 8 / 4, so also the lpb input rings' 128 / 256), before the same boundary four chunks on (the ring wraps
    there and is read through its head mirror) and five chunks on; and 64 + k bytes before them, where the group fast
    path's window (DEC_AHEAD = 64) crosses the boundary.  Dense sequences follow, so later headers take further phases."""
    for B in (128, 256, 512, 1024):
        for j in (1, 4, 5):
            for back in (0, 64):
                for k in range(9):
                    target = B * j - back - k                  # stream position of the second header
                    # first sequence: L literals and a match of 4 or 19 (one more header byte), whichever lands exactly
                    L, mlen = next((L, m) for L in range(target, 0, -1) for m in (4, 19) if L + header_size(L, m) == target)
                    seqs = [(g.lits(L), 3, mlen)] + _dense(g, 40)
                    g.add(f"place/B{B}/j{j}/back{back}/k{k}", seqs, g.lits(16 + 8 * (k % 3)))
    # op crossing cap - 112, where the group fast path hands over to the careful one (cap = n, n + 1)
    for d in range(-4, 9):
        for mlen in (4, 30, 64):
            seqs = g.prefix(300) + [(g.lits(20), 9, mlen)]
            rest = 112 + d - 20 - mlen
            tail = []
            while rest > 20 + 12:
                tail.append((g.lits(5), 11, 15)); rest -= 20
            g.add(f"place/out-fast/d{d}/M{mlen}", seqs + tail, g.lits(rest), (0, 1))


# pools of the random mixes: lengths at the thresholds above, and some arbitrary ones
_LIT_POOL = (0, 1, 2, 3, 4, 7, 8, 14, 15, 16, 17, 31, 32, 33, 63, 64, 65, 269, 270, 271, 525)
_MATCH_POOL = (4, 5, 6, 7, 8, 18, 19, 20, 31, 32, 33, 64, 65, 66, 248, 249, 273, 274, 275, 505)
_OFF_POOL = (1, 2, 3, 4, 5, 6, 7, 8, 31, 32, 33, 63, 64, 65, 128, 248, 249, 252, 256, 257, 504, 505, 512, 1024, 4096)


def _mix(g, n):
    """Sequences drawn from the pools until the block holds about n bytes, then 5-100 last literals."""
    rng = g.rng
    seqs, op = [], 0
    while op < n:
        L = int(rng.choice(_LIT_POOL)) if rng.random() < 0.9 else int(rng.integers(0, 3000))
        if op + L == 0:
            L = 1
        mlen = int(rng.choice(_MATCH_POOL)) if rng.random() < 0.9 else int(rng.integers(4, 5000))
        c = rng.random()
        if c < 0.6:
            off = int(rng.choice(_OFF_POOL))
        elif c < 0.75:
            off = L + int(rng.integers(-1, 2))
        elif c < 0.8:
            off = op + L
        else:
            off = int(rng.integers(1, 65536))
        off = max(1, min(off, op + L, 65535))
        seqs.append((g.lits(L), off, mlen))
        op += L + mlen
    return seqs, g.lits(int(rng.choice((5, 6, 7, 8, 9, 11, 12, 13, 16, 64, 100))))


def _random(g):
    sizes = [13, 20, 40, 64, 100, 200, 500, 1000, 3000, 5000, 20_000] * 6 + [65_536, 100_000, 200_000]
    for i, n in enumerate(sizes):
        seqs, last = _mix(g, n)
        g.add(f"mix/{i}/n{n}", seqs, last, (0,))


def _perturb(g):
    """Truncation by 1-8 bytes, one appended byte (0 or 0xFF), cap +- k -- on a sample of the cases above."""
    rng = g.rng
    base = list(g.cases)
    picks = rng.choice(len(base), size=400, replace=False)
    for i in sorted(int(p) for p in picks):
        c = base[i]
        kind = i % 4
        if kind == 0:
            k = 1 + i % 8
            g.cases.append(Case(f"{c.name}/cut{k}", c.stream[:-k], c.cap))
        elif kind == 1:
            g.cases.append(Case(f"{c.name}/append{'ff' if i & 4 else '00'}", c.stream + (b"\xff" if i & 4 else b"\x00"), c.cap))
        else:
            d = int(rng.integers(1, 14)) * (1 if kind == 2 else -1)
            g.cases.append(Case(f"{c.name}/cap{d:+d}", c.stream, c.cap + d))


def corpus(seed: int = 1):
    """The constructed cases, in a fixed order: a pure function of `seed`."""
    g = _Gen(seed)
    for family in (_tail, _offsets, _ring_window, _lengths, _placement, _random, _perturb):
        family(g)
    names = [c.name for c in g.cases]
    assert len(set(names)) == len(names)
    return g.cases
