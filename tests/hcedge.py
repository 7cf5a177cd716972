"""Constructed LZ4HC blocks at the edges of the warp encoders' search, literal scan and window -- TEST INFRASTRUCTURE ONLY.

The reference's chain walk from q (original/lz4hc.c:394-518) visits the positions below q with q's 15-bit hash in
descending order, then position 0, and examines at most 256 of them -- 257 when the first lies within 4 bytes of q (the
repeat detector consumes it without an attempt).  Content reaches the ends of that only by chance, so the blocks here are
noise with chosen words planted at chosen places of a walk: the word searched, copies of it that match for a chosen
length, and "colliders" -- other words with the same hash, which fill the bucket and spend attempts without matching.

The noise is cleaned until no 4-byte window that holds a noise byte repeats anywhere in the block or falls into a bucket
of a planted window: the planted structure is the only structure.  Each builder then checks what it built twice -- the
walk place of every planted candidate from the bytes, and the sequence the port oracle emits at the searched position
(offset and length, read back with sequences()) -- so a builder that misses its threshold fails loudly instead of adding
one more block that merely agrees byte for byte.

A case says whether the warp kernels (lz4hc_warp.cuh, lz4hc_window.cuh) must encode it or hand it back (HCW_FALLBACK).
catalogue(seed) is a pure function of its seed; tests/golden/hc_constructed_v1.json holds what the reference returned on
it (tests/golden/make_golden.py).
"""
from __future__ import annotations

import functools
from typing import NamedTuple

import numpy as np

MULT = 2654435761
MULT_INV = pow(MULT, -1, 1 << 32)
K = 256                                               # MAX_NB_ATTEMPTS (original/lz4hc.c:184)


class Case(NamedTuple):
    name: str
    data: bytes
    warp: bool                                        # True: the warp kernels encode it; False: they hand it back


def hash15(w):
    """LZ4HC's hash of little-endian 4-byte words (a scalar or a uint32 array)."""
    return ((np.asarray(w, np.uint64) * MULT) & 0xFFFFFFFF) >> 17


def words(d) -> np.ndarray:
    a = np.frombuffer(bytes(d), np.uint8).astype(np.uint32) if not isinstance(d, np.ndarray) else d.astype(np.uint32)
    return a[:-3] | (a[1:-2] << 8) | (a[2:-1] << 16) | (a[3:] << 24)


def word_bytes(w: int) -> bytes:
    return int(w).to_bytes(4, "little")


def walk(d: bytes, q: int) -> list:
    """The reference's walk from q in a block of at most 64 KiB, before any place is dropped by the attempt budget: the
    positions 1..q-1 with q's hash, nearest first, then position 0."""
    h = hash15(words(d))
    return [int(p) for p in (np.flatnonzero(h[1:q] == h[q]) + 1)[::-1]] + [0]


def sequences(comp: bytes) -> list:
    """An LZ4 block's sequences as (position of the match, literal length, offset, match length)."""
    out, i, pos = [], 0, 0
    while i < len(comp):
        tok = comp[i]; i += 1
        L = tok >> 4
        if L == 15:
            while True:
                b = comp[i]; i += 1; L += b
                if b != 255:
                    break
        i += L; pos += L
        if i >= len(comp):
            break
        off = comp[i] | comp[i + 1] << 8; i += 2
        M = tok & 15
        if M == 15:
            while True:
                b = comp[i]; i += 1; M += b
                if b != 255:
                    break
        out.append((pos, L, off, M + 4)); pos += M + 4
    return out


def _seqs(d):
    import oracle
    r, o = oracle.encode_hc(d)
    assert r > 0
    return sequences(o)


def at(seqs, q):
    """The sequence whose match starts at q, or None."""
    for s in seqs:
        if s[0] == q:
            return s
    return None


def offsets(seqs):
    return {s[2] for s in seqs}


class _Block:
    """Noise with planted bytes; done() cleans the noise (see the module's docstring)."""

    def __init__(self, n, rng):
        self.rng = rng
        self.d = rng.integers(0, 256, n, dtype=np.uint8)
        self.fixed = np.zeros(n, bool)

    def put(self, p, b, over=False) -> int:
        """Plants b at p; over: b may overwrite earlier plants."""
        b = np.frombuffer(bytes(b), np.uint8)
        assert p >= 0 and p + len(b) <= len(self.d)
        assert over or not (self.fixed[p:p + len(b)] & (self.d[p:p + len(b)] != b)).any(), "plants overlap"
        self.d[p:p + len(b)] = b
        self.fixed[p:p + len(b)] = True
        return p + len(b)

    def done(self) -> bytes:
        d, f = self.d, self.fixed
        wfixed = f[:-3] & f[1:-2] & f[2:-1] & f[3:]
        for _ in range(400):
            w = words(d)
            h = hash15(w)
            _, inv, cnt = np.unique(w, return_inverse=True, return_counts=True)
            bad = ~wfixed & ((cnt[inv] > 1) | np.isin(h, np.unique(h[wfixed])))
            if not bad.any():
                return d.tobytes()
            for i in np.flatnonzero(bad):
                free = np.flatnonzero(~f[i:i + 4])
                d[i + free[self.rng.integers(len(free))]] = self.rng.integers(0, 256)
        raise AssertionError("noise did not clean up")


class _Gen:
    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.cases = []

    def bytes(self, n) -> bytes:
        return self.rng.integers(0, 256, n, dtype=np.uint8).tobytes()

    def word(self) -> int:
        while True:
            w = int(self.rng.integers(0, 1 << 32))
            b = word_bytes(w)
            if len(set(b)) == 4:
                return w

    def after(self, w: int, n: int) -> bytes:
        """n random bytes to follow the word w: no window of w + them but the first has w's hash."""
        while True:
            b = self.bytes(n)
            if not (hash15(words(word_bytes(w) + b))[1:] == hash15(w)).any():
                return b

    def colliders(self, w: int, count: int) -> list:
        """`count` distinct words other than w with w's hash, as bytes."""
        h = int(hash15(w))
        out, seen = [], {w}
        while len(out) < count:
            c = (MULT_INV * ((h << 17) | int(self.rng.integers(0, 1 << 17)))) & 0xFFFFFFFF
            if c not in seen and len(set(word_bytes(c))) == 4:
                seen.add(c); out.append(word_bytes(c))
        assert all(int(hash15(int.from_bytes(c, "little"))) == h for c in out)
        return out

    def plant_colliders(self, b: _Block, at: int, cs) -> int:
        """The colliders one noise byte apart from `at` on; returns the position behind the last."""
        for c in cs:
            at = b.put(at, c) + 1
        return at

    def add(self, name, data, warp=True):
        self.cases.append(Case(name, data, warp))


def _check_walk(d, q, want: dict):
    """want: {position: place in q's walk}."""
    wk = walk(d, q)
    for p, k in want.items():
        assert p in wk and wk.index(p) == k, (p, k, wk.index(p) if p in wk else None)


# ---- the attempt budget in the search -----------------------------------------------------------------------------
SEARCH_PLACES = (30, 31, 32, 33, 62, 63, 64, 65, 126, 127, 128, 129, 254, 255, 256)


def _search_budget(g: _Gen):
    """q's walk: a short equal candidate s at place 0 (W + 1 byte), colliders, then a long one p (W + 40 bytes) at place P.
    The search takes p while P < K.  From P = K on it takes s, and the wider search at q + 3 (start_limit q + 1) then
    finds p + 1 and moves the match to q + 1 (the scan hits at q either way)."""
    for P in SEARCH_PLACES:
        W, X = g.word(), g.bytes(40)
        cs = g.colliders(W, P - 1)
        b = _Block(64 + 44 + 20 + 5 * len(cs) + 60 + 44 + 64, g.rng)
        p = 64
        b.put(p, word_bytes(W) + X)
        s = g.plant_colliders(b, p + 44 + 20, cs) + 10
        b.put(s, word_bytes(W) + X[:1])
        q = s + 50
        b.put(q, word_bytes(W) + X)
        d = b.done()
        _check_walk(d, q, {s: 0, p: P})
        seqs = _seqs(d)
        if P < K:
            assert at(seqs, q)[2:] == (q - p, 44), (P, seqs)
        else:
            assert at(seqs, q) is None and at(seqs, q + 1)[2:] == (q - p, 43), (P, seqs)
        g.add(f"search-budget-place{P}", d)


def _search_budget_repeat(g: _Gen):
    """The budget of 257 through the repeat detector: W at r = q - delta and at q (delta = 4: a period-4 run, so r is
    candidate 0 and costs no attempt), 255 colliders, then the long candidate p at place 256.  r itself is matched to p
    first (its match ends at r + 4), so the scan resumes at q.  delta = 4 takes p; delta = 5 (not a repeat) takes r,
    and the wider search at q + 2 moves the match to p + 1."""
    for delta in (4, 5):
        W, X = g.word(), g.bytes(40)
        cs = g.colliders(W, 255)
        b = _Block(64 + 44 + 20 + 5 * 255 + 60 + 4 + delta + 44 + 64, g.rng)
        p = 64
        b.put(p, word_bytes(W) + X)
        r = g.plant_colliders(b, p + 44 + 20, cs) + 10
        b.put(r, word_bytes(W))
        q = r + delta
        b.put(q, word_bytes(W) + X)
        d = b.done()
        assert d[q + 4] != d[r + 4] and d[r + 4] != d[p + 4]
        _check_walk(d, q, {r: 0, p: 256})
        seqs = _seqs(d)
        assert at(seqs, r)[2:] == (r - p, 4)
        if delta == 4:
            assert at(seqs, q)[2:] == (q - p, 44), (delta, seqs)
        else:                                           # (r taken, then moved to q + 1 as in _search_budget)
            assert at(seqs, q) is None and at(seqs, q + 1)[2:] == (q - p, 43), (delta, seqs)
        g.add(f"search-budget-repeat-delta{delta}", d)


# ---- the attempt budget in the literal scan ------------------------------------------------------------------------
def _scan_budget(g: _Gen):
    """q's only equal candidate p (W + 40 bytes) at place P behind colliders: the scan hits at q while P < K, else q stays
    a literal and q + 1 takes the match.  near = a collider at q - 4 (candidate 0, free: K = 257) or at q - 5 (K = 256),
    the equal candidate at place 256."""
    for P, near in ((254, 0), (255, 0), (256, 0), (256, 4), (256, 5)):
        W, X = g.word(), g.bytes(40)
        cs = g.colliders(W, P)
        far = cs[:-1] if near else cs
        b = _Block(64 + 44 + 20 + 5 * len(cs) + 60 + 44 + 64, g.rng)
        p = 64
        b.put(p, word_bytes(W) + X)
        q = g.plant_colliders(b, p + 44 + 20, far) + 40
        if near:
            b.put(q - near, cs[-1])
        b.put(q, word_bytes(W) + X)
        d = b.done()
        _check_walk(d, q, {p: P} if not near else {p: P, q - near: 0})
        K_ = K + 1 if near == 4 else K
        seqs = _seqs(d)
        if P < K_:
            assert at(seqs, q)[2] == q - p, (P, near)
        else:
            assert at(seqs, q) is None and at(seqs, q + 1)[2] == q - p, (P, near)
        g.add(f"scan-budget-place{P}" + (f"-near{near}" if near else ""), d)


# ---- position 0, the walk's last candidate -------------------------------------------------------------------------
def _position_zero(g: _Gen):
    """The block starts with q's bytes, D entries of q's bucket in front of it: position 0 is place D.  scan: nothing else
    matches (taken iff D < K: else q + 1 matches position 1).  search: a short candidate at place 0 makes the scan hit
    either way, and the search takes position 0 iff D < K."""
    for kind, depths in (("scan", (0, 254, 255, 256)), ("search", (1, 254, 255, 256))):
        for D in depths:
            W, X = g.word(), g.bytes(40)
            cs = g.colliders(W, D - (kind == "search"))
            b = _Block(44 + 20 + 5 * len(cs) + 60 + 44 + 64, g.rng)
            b.put(0, word_bytes(W) + X)
            q = g.plant_colliders(b, 44 + 20, cs) + 10
            s = None
            if kind == "search":
                s = q
                b.put(s, word_bytes(W) + X[:1])
                q += 40
            b.put(q, word_bytes(W) + X)
            d = b.done()
            _check_walk(d, q, {0: D, **({s: 0} if s is not None else {})})
            seqs = _seqs(d)
            if D < K:
                assert at(seqs, q)[2:] == (q, 44), (kind, D)
            else:                                       # (search: s taken, then moved to q + 1 as in _search_budget)
                assert at(seqs, q) is None and at(seqs, q + 1)[2:] == (q, 43), (kind, D)
            g.add(f"pos0-{kind}-depth{D}", d)


# ---- ties: the first maximum wins ----------------------------------------------------------------------------------
TIE_PLACES = ((0, 1), (3, 17), (30, 31), (31, 32), (63, 64), (127, 128), (5, 200))


def _ties(g: _Gen):
    """Two candidates matching for the same length at places a < b: the search takes a.  One more equal byte at b: b."""
    for a, bb in TIE_PLACES:
        for longer in (False, True):
            W, X = g.word(), g.bytes(30)
            cs = g.colliders(W, bb - 1)
            blk = _Block(64 + 5 * len(cs) + 3 * 60 + 3 * 44 + 64, g.rng)
            pb = 64
            blk.put(pb, word_bytes(W) + X[:20 + longer])
            pa = g.plant_colliders(blk, pb + 40, cs[:bb - a - 1]) + 10
            blk.put(pa, word_bytes(W) + X[:20])
            q = g.plant_colliders(blk, pa + 40, cs[bb - a - 1:]) + 10
            blk.put(q, word_bytes(W) + X)
            d = blk.done()
            _check_walk(d, q, {pa: a, pb: bb})
            seq = at(_seqs(d), q)
            assert seq[2:] == ((q - pb, 25) if longer else (q - pa, 24)), (a, bb, longer, seq)
            g.add(f"tie-search-{a}-{bb}" + ("-deeper-longer" if longer else ""), d)


def _wider_ties(g: _Gen):
    """The wider search at wq = q + ml - 2 (start_limit q + 1) behind a first match of ml = 24 at q: candidates c1 (place 0)
    and c2 (place 1, or 32 behind colliders) with different backward extensions.  Tie: c1 (4 back, 24 forward) and c2
    (12 back, 16 forward) reach 28, c1 is taken.  Deeper longer: c1 (12 + 15) reaches 27, c2 (4 + 24) 28, c2 is taken.
    The winner's copy runs to the end of q's bytes, so no later search finds a longer one."""
    for cross in (False, True):
        for longer in (False, True):
            U, T = g.bytes(24), g.bytes(22)
            ml = len(U)
            cs = g.colliders(int.from_bytes(U[ml - 2:] + T[:2], "little"), 31 if cross else 0)
            blk = _Block(64 + 5 * len(cs) + 4 * 80 + 64, g.rng)

            def cand(at, back, t):                      # back bytes before wq, then U's last 2 bytes and t of T
                blk.put(at, U[ml - 2 - back:] + T[:t])
                return at + back
            c2 = cand(64, 4, 22) if longer else cand(64, 12, 14)
            at_ = g.plant_colliders(blk, c2 + 40, cs) + 10
            c1 = cand(at_, 12, 13) if longer else cand(at_, 4, 22)
            s = c1 + 50
            blk.put(s, U)
            q = s + 40
            blk.put(q, U + T)
            d = blk.done()
            wq = q + ml - 2
            _check_walk(d, wq, {c1: 0, c2: 32 if cross else 1})
            seqs = _seqs(d)
            assert at(seqs, q)[2] == q - s
            want, other = (wq - c2, wq - c1) if longer else (wq - c1, wq - c2)
            assert want in offsets(seqs) and other not in offsets(seqs), (cross, longer, seqs)
            g.add(f"tie-wider-{'cross' if cross else 'same'}-batch" + ("-deeper-longer" if longer else ""), d)


# ---- length counting -----------------------------------------------------------------------------------------------
FORWARD_COMMON = (124, 127, 128, 129, 131, 132, 255, 256, 257)


def _forward_lengths(g: _Gen):
    """A match of 4 + c bytes (c = the common length after the word, around the 128-byte steps of the warp count), p the
    only equal candidate of its batch ("single") or with a 5-byte one beside it ("multi")."""
    for c in FORWARD_COMMON:
        for multi in (False, True):
            W, Y = g.word(), g.bytes(c + 30)
            blk = _Block(64 + 2 * (c + 40) + 60 + 64, g.rng)
            p = 64
            blk.put(p, word_bytes(W) + Y[:c])
            q = p + c + 40
            if multi:
                blk.put(q, word_bytes(W) + Y[:1])
                q += 20
            blk.put(q, word_bytes(W) + Y)
            d = blk.done()
            _check_walk(d, q, {p: 1 if multi else 0})
            assert at(_seqs(d), q)[2:] == (q - p, 4 + c), (c, multi)
            g.add(f"forward-{4 + c}-{'multi' if multi else 'single'}", d)


MATCHLIMIT_LENGTHS = (36, 37, 38, 39, 132, 133, 134, 135)


def _matchlimit(g: _Gen):
    """The match at q runs into matchlimit = n - 5 (the block ends there: every residue of (matchlimit - q) mod 4), or
    stops one byte short of it; p's copy goes on past the block's end, so only the limit stops the count."""
    for L in MATCHLIMIT_LENGTHS:
        for short in (False, True):
            for multi in (False, True):
                W = g.word()
                tail = g.after(W, L + 1 + 8)                   # d[q + 4 : n], then 8 more bytes in p's copy
                n = 64 + (L + 20) + 60 + (20 if multi else 0) + L + 5
                q = n - 5 - L
                blk = _Block(n, g.rng)
                p = 64
                cp = bytearray(word_bytes(W) + tail)
                tail = tail[:L + 1]
                if short:
                    cp[L - 1] ^= 0x5A
                blk.put(p, bytes(cp))
                if multi:
                    blk.put(q - 20, word_bytes(W) + tail[:1])
                blk.put(q, word_bytes(W) + tail)
                d = blk.done()
                assert len(d) - 5 - q == L
                _check_walk(d, q, {p: 1 if multi else 0})
                assert at(_seqs(d), q)[2:] == (q - p, L - short), (L, short, multi)
                g.add(f"matchlimit-{L}" + ("-short" if short else "") + ("-multi" if multi else "-single"), d)


BACK = (3, 4, 5, 31, 32, 33)


def _backward(g: _Gen):
    """Backward extension in the wider search at wq = q + ml - 2 behind a first match at q (from s at q's place 0), of
    b bytes, stopped
    * "limit": by start_limit = q + 1 (ml = b + 3).  The byte in front of it matches too: the copy there is a candidate
      of q, hidden from q's search at place 256 behind colliders;
    * "ref0": by the reference reaching position 0 (the candidate is position b).  ml = b + 20 puts the wider match's
      start 18 bytes behind q, where the look-ahead keeps it as found.
    "multi" adds a second, shorter equal candidate to c's batch."""
    for stop in ("limit", "ref0"):
        for bk in BACK:
            for multi in (False, True):
                ml = bk + 3 if stop == "limit" else bk + 20
                fwd = 12 if stop == "limit" else 24
                U, T = g.bytes(ml), g.bytes(40)
                Vw = int.from_bytes(U[ml - 2:] + T[:2], "little")
                cu = g.colliders(int.from_bytes(U[:4], "little"), 255) if stop == "limit" else []
                blk = _Block(80 + 5 * len(cu) + 6 * (ml + 60) + 64, g.rng)
                if stop == "ref0":
                    c = bk
                    blk.put(0, U[ml - 2 - bk:] + T[:fwd])
                    at_ = c + 2 + fwd + 40
                else:
                    hide = 64                                  # U from q's start on: q's candidate at place 256
                    blk.put(hide, U + T[:fwd])
                    c = hide + ml - 2
                    at_ = g.plant_colliders(blk, c + 2 + fwd + 20, cu) + 10
                c2 = None
                if multi:
                    c2 = at_
                    blk.put(c2, U[ml - 2:] + T[:2])
                    at_ += 30
                s = at_
                blk.put(s, U)
                q = s + ml + 30
                blk.put(q, U + T)
                d = blk.done()
                wq = q + ml - 2
                _check_walk(d, wq, {c: 1 if multi else 0, **({c2: 0} if multi else {})})
                if stop == "limit":
                    _check_walk(d, q, {s: 0, c - ml + 2: 256})
                seqs = _seqs(d)
                assert at(seqs, q) is None or at(seqs, q)[2] == q - s
                # the wider match, b bytes in front of wq
                assert any(x[0] == wq - bk and x[2] == wq - c for x in seqs), (stop, bk, multi, seqs)
                g.add(f"back-{stop}-{bk}-{'multi' if multi else 'single'}", d)


# ---- the repeat detector -------------------------------------------------------------------------------------------
def colliding_triple() -> bytes:
    """Three bytes whose period-3 run has two words in one bucket (and a third in another): the repeat detector's chain is
    then not the static one, and the warp kernels hand the block back."""
    for a in range(1, 256):
        for b in range(a + 1, 256):
            for c in range(b + 1, 256):
                s0, s1, s2 = bytes([a, b, c, a]), bytes([b, c, a, b]), bytes([c, a, b, c])
                if hash15(int.from_bytes(s1, "little")) == hash15(int.from_bytes(s2, "little")) and \
                        hash15(int.from_bytes(s0, "little")) != hash15(int.from_bytes(s1, "little")):
                    return bytes([a, b, c])
    raise AssertionError


def _period(g: _Gen, delta: int) -> bytes:
    """A period of delta bytes whose delta rotations (the run's words) have distinct hashes."""
    while True:
        u = g.bytes(delta)
        if len(set(u)) < delta:
            continue
        run = u * (8 // delta + 1)
        if len({int(hash15(int.from_bytes(run[i:i + 4], "little"))) for i in range(delta)}) == delta:
            return u


def _repeats(g: _Gen):
    """Runs of period 1..4 whose words do not share a bucket: the repeat detector's chain is the static one, so the warp
    kernels encode them.  The match at q0 + delta (offset delta) has ml = R - delta; R moves the run's end across the
    wider search at ip + ml - 2.  "copy": an earlier copy of the run and 8 more bytes beats the repeat.  The colliding
    triple (two of its words share a bucket) is handed back."""
    for delta in (1, 2, 3, 4):
        for R in (delta + 4, delta + 5, delta + 6, delta + 7, 40):
            for copy in ((False, True) if R == 40 else (False,)):
                u = _period(g, delta)
                run = (u * (R // delta + 1))[:R]
                tail = g.bytes(8)
                blk = _Block(64 + 2 * (R + 50) + 64, g.rng)
                if copy:
                    blk.put(64, run + tail)
                q0 = 64 + R + 50
                blk.put(q0, run + (tail if copy else b""))
                d = blk.done()
                seq = at(_seqs(d), q0 + (0 if copy else delta))
                if copy:
                    assert seq[2:] == (q0 - 64, R + 8), (delta, seq)
                else:
                    assert seq[2:] == (delta, R - delta), (delta, R, seq)
                g.add(f"repeat-period{delta}-run{R}" + ("-copy" if copy else ""), d)
    t = colliding_triple()
    for R in (30, 300):
        blk = _Block(64 + R + 64, g.rng)
        blk.put(64, (t * R)[:R])
        d = blk.done()
        assert at(_seqs(d), 67)[2] == 3
        g.add(f"repeat-colliding-triple-run{R}", d, warp=False)


# ---- blocks above 64 KiB: the window -------------------------------------------------------------------------------
WINDOW_Q = (65536 + 40, 131072, 131072 + 3, 196608 - 1, 196608 + 17)
MARK = b"\x01WINDOWEDGE\x02"
# the marks behind q, farthest first, each written over the ones before it, then q's own
WINDOW_MARKS = ((65535,), (65536,), (65536 + 65535, 65536), (65536 + 65536, 65536), (65537, 1), (70000, 65535, 65534))


def _covering(seqs, q):
    return [s for s in seqs if s[0] <= q < s[0] + s[3]]


def _window_edges(g: _Gen):
    """The same 12 bytes at q and at chosen distances behind it, q on and across the 64 KiB segment boundaries.  A mark
    whose 12 bytes survive and which lies at most 65535 back is a candidate; q takes the nearest (the marks tie), and
    with none q stays a literal.  So a mark 65535 back is taken, one 65536 back is not; a bucket whose previous position
    lies 65536 back has that delta clamped to 65535 (pointing into noise) and its walk ends; a mark 65537 back behind an
    overwritten one 1 back gives nothing; of the marks 65535 and 65534 back, only the second survives."""
    for q in WINDOW_Q:
        for back in WINDOW_MARKS:
            marks = [q - b for b in back]
            if min(marks) < 1:
                continue
            blk = _Block(q + 3000, g.rng)
            for m in marks + [q]:
                blk.put(m, MARK, over=True)
            d = blk.done()
            live = [m for m in marks if d[m:m + 12] == MARK and q - m <= 65535]
            seqs = _seqs(d)
            if live:
                assert at(seqs, q)[2] == q - max(live), (q, back)
            else:
                assert not _covering(seqs, q), (q, back)
            g.add(f"window-q{q}-" + "-".join(map(str, back)), d)


def _window_position_zero(g: _Gen):
    """q's bytes at position 0 and an empty bucket: position 0 is the walk's last candidate for q = 65535 and out of the
    window for q = 65536."""
    for q in (65535, 65536):
        blk = _Block(q + 3000, g.rng)
        blk.put(0, MARK); blk.put(q, MARK)
        d = blk.done()
        s = at(_seqs(d), q)
        assert (s[2] == q) if q < 65536 else s is None, (q, s)
        g.add(f"window-pos0-q{q}", d)


def _window_skips(g: _Gen):
    """Runs of 100-300 KiB inside text: one match crosses a segment boundary, or covers whole segments, which no search
    ever needs and so are never indexed."""
    from tests import cases
    t = cases.content("mixed", 30000, seed=5).tobytes()
    for run, whole in ((100_000, 0), (300_000, 4)):
        d = t + bytes(run) + t[::-1] + bytes([7]) * (run // 2) + t
        z = [s for s in _seqs(d) if s[2] == 1 and s[0] <= 30004 and s[0] + s[3] >= 30000 + run]
        assert len(z) == 1, run
        a, e = z[0][0], z[0][0] + z[0][3]
        assert a < 65536 < e and sum(a <= k << 16 and (k + 1) << 16 <= e for k in range(1, len(d) >> 16)) == whole, run
        g.add(f"window-skip-run{run}", d)


def _window_one_bucket(g: _Gen):
    """Zeros over three segments: the one match runs from position 1 to matchlimit.  Zeros to 200000, then text: the
    search behind the zeros lies in segment 3, so segment 2 is indexed with all 65536 of its positions in one bucket (the
    bucket end that needs the u32 `end`)."""
    from tests import cases
    d = bytes(196608 + 4000)
    assert at(_seqs(d), 1) == (1, 1, 1, len(d) - 6)
    g.add("window-one-bucket-zeros", d)
    d = bytes(200000) + cases.content("mixed", 5000, seed=3).tobytes()
    s = at(_seqs(d), 1)
    assert s[2] == 1 and 196608 < s[0] + s[3] < 262144, s
    g.add("window-one-bucket-then-text", d)


def _window_repeats(g: _Gen):
    """Runs of period 1..4 over 200000 bytes, past a segment: the repeat detector's run is longer than a segment and its
    chain writes wrap the u16 table; the warp kernels still encode them.  The colliding triple past 64 KiB is handed back,
    the same run of a triple that does not collide is encoded."""
    for period in (1, 2, 3, 4):
        L = 200000 // period * period
        blk = _Block(3000 + L + 3000, g.rng)
        blk.put(3000, bytes(range(10, 10 + period)) * (L // period))
        d = blk.done()
        assert at(_seqs(d), 3000 + period)[2:] == (period, L - period), period
        g.add(f"window-repeat-period{period}", d)
    for t, warp in ((colliding_triple(), False), (bytes([1, 2, 3]), True)):
        blk = _Block(70000 + 600 + 500, g.rng)
        blk.put(70000, t * 200)
        d = blk.done()
        assert at(_seqs(d), 70003)[2:] == (3, 597)
        g.add("window-colliding-triple" if not warp else "window-triple-not-colliding", d, warp=warp)


@functools.lru_cache(maxsize=2)
def window_cases(seed: int = 1) -> tuple:
    """The cases above 64 KiB (the window kernel's), in a fixed order."""
    g = _Gen([seed, 65536])
    for build in (_window_edges, _window_position_zero, _window_skips, _window_one_bucket, _window_repeats):
        build(g)
    return tuple(g.cases)


def catalogue(seed: int = 1) -> list:
    """Every constructed case, in a fixed order: the blocks of at most 64 KiB, then window_cases(seed)."""
    g = _Gen(seed)
    for build in (_search_budget, _search_budget_repeat, _scan_budget, _position_zero, _ties, _wider_ties,
                  _forward_lengths, _matchlimit, _backward, _repeats):
        build(g)
    cases = g.cases + list(window_cases(seed))
    names = [c.name for c in cases]
    assert len(set(names)) == len(names)
    return cases
