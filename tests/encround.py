"""A model of the fast encoder's parse (lz4net_b200/csrc/lz4_encode.cuh) for constructed-block tests.

parse() is the reference's serial greedy parse (LZ4_compress64kCtx / LZ4_compressCtx, no output limit).  Besides the
sequences it records every find-match loop: what started it, the attempt number and position of each of its probes and
how it ended.  rounds() maps those loops onto the kernel's rounds for one variant and EncTune: which serial iterations
one round evaluates at once, which of them share a hash bucket, where its first event f falls and which path of
find_round resolves the sharing.  counts() sums that up in the kernel's event counters (enc_prof.cuh).

The kernel's state machine, as modelled here:
  * a loop starts at attempt 67 (findMatchAttempts) at the block start and after a post-match probe tried alone that
    missed; its first round is 32 iterations wide;
  * after a match with literal run L (before the catch-up) the post-match probe is tried alone when L < probe_max;
    otherwise it rides in a fused round from attempt 65 (lane 0 inserts ip-2, lane 1 probes ip), 64 wide when
    L >= wide_min;
  * every round after one without an event is 64 wide; variant 1 is never wide.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

LIMIT64K = 65547
MULT = 2654435761
MULT_INV = pow(MULT, -1, 1 << 32)
TUNE = (12, 8, 24)                                    # EncTune: lane_copy_max, probe_max, wide_min


def shift_of(n: int) -> int:
    return 20 if n >= LIMIT64K else 19


def hash_of(w: int, shift: int) -> int:
    return ((w * MULT) & 0xFFFFFFFF) >> shift


def word_with_hash(bucket: int, shift: int, low: int) -> int:
    """The word whose hash is `bucket`, with `low` (< 2**shift) as the low bits of its product: the multiplier is odd."""
    return (MULT_INV * ((bucket << shift) | low)) & 0xFFFFFFFF


@dataclass
class Loop:
    """One find-match loop of the serial parse and the post-match probe in front of it.
    after: index of the sequence it follows (-1: block start); m: that sequence's match end; L: its literal run as
    found (before the catch-up); post_hit: the post-match probe at m hit (then the loop has no probes);
    probes: (attempt, position) of each probe, from attempt 67; end: 'hit' (the last probe hit), 'finish' (the
    iteration of attempt end_attempt ran past mflimit) or 'post' (the post-match probe hit)."""
    after: int
    m: int
    L: int
    post_hit: bool
    probes: list = field(default_factory=list)
    end: str = ""
    end_attempt: int = 0


@dataclass
class Parse:
    seqs: list      # (anchor, ip found, ip caught up, ref caught up, match end)
    probes: list    # positions probed by the find-match loops, in order
    last: int       # anchor of the last literals
    loops: list     # Loop records, in order
    refs: dict = field(default_factory=dict)      # position: the table's candidate when it was last probed


def parse(d: bytes) -> Parse:
    n = len(d)
    general = n >= LIMIT64K
    shift = shift_of(n)
    table = [0] * (1 << (32 - shift))
    mv = memoryview(d)

    def word(p):
        return int.from_bytes(mv[p:p + 4], "little")

    def h(p):
        return ((word(p) * MULT) & 0xFFFFFFFF) >> shift

    def hit(ref, ip):
        return (not general or ref > ip - 65536) and word(ref) == word(ip)

    seqs, probes, loops, refs = [], [], [], {}
    if n < 13:
        return Parse(seqs, probes, 0, loops)
    mflimit, matchlimit = n - 12, n - 5
    anchor = 0
    table[h(0)] = 0
    ip = 1
    lp = Loop(-1, 0, 0, False)
    while True:
        loops.append(lp)
        attempts, fwd = 67, ip
        while True:
            ip = fwd
            step = attempts >> 6
            attempts += 1
            fwd = ip + step
            if fwd > mflimit:
                lp.end, lp.end_attempt = "finish", attempts - 1
                return Parse(seqs, probes, anchor, loops, refs)
            k = h(ip); ref = table[k]; table[k] = ip
            refs[ip] = ref
            probes.append(ip)
            lp.probes.append((attempts - 1, ip))
            if hit(ref, ip):
                lp.end, lp.end_attempt = "hit", attempts - 1
                break
        found = ip
        while ip > anchor and ref > 0 and d[ip - 1] == d[ref - 1]:
            ip -= 1; ref -= 1
        while True:
            m, r = ip + 4, ref + 4
            while m < matchlimit and d[m] == d[r]:
                m += 1; r += 1
            seqs.append((anchor, found, ip, ref, m))
            L = found - seqs[-1][0]
            anchor = m
            if m > mflimit:
                return Parse(seqs, probes, anchor, loops, refs)
            table[h(m - 2)] = m - 2
            k = h(m); ref = table[k]; table[k] = m
            refs[m] = ref
            if hit(ref, m):
                loops.append(Loop(len(seqs) - 1, m, L, True, end="post", end_attempt=66))
                ip = found = m
                continue
            break
        lp = Loop(len(seqs) - 1, m, L, False)
        ip = m + 1


def position(org: int, a: int) -> int:
    """Position of attempt a (>= 65) of a loop whose attempt 67 sits at org + 3: org + S(a), S(a) = sum_{j<a} (j >> 6)."""
    q = a >> 6
    return org + q * (32 * (q - 1) + (a & 63))


@dataclass
class Round:
    """One round of find_round.  Indices are the round's iterations 0 .. 32*W-1 (lane l: l and 32 + l)."""
    loop: int           # index into Parse.loops
    k: int              # round number inside its loop
    A0: int             # attempt of iteration 0
    W: int
    fused: bool
    simple: bool
    org: int
    pos: list           # position of every iteration
    valid: list         # valid iterations are a prefix (fused lanes 0 and 1 always are)
    hashes: list        # hash of every valid iteration (None for invalid ones)
    groups: list        # sharer groups: sorted index lists of >= 2 valid iterations with one hash, by first index
    f: int              # first event (hit or first invalid iteration); 32*W: none in this round
    event: str          # 'hit', 'finish' or '' (none)
    path: str           # 'exact', 'pair' or 'none' (no sharing: the pair path's code with nothing to resolve)

    @property
    def nv(self):
        return sum(self.valid)


@dataclass
class Probe:
    """A post-match probe tried alone (probe_first): insert m-2, probe m."""
    loop: int
    m: int
    hit: bool


def rounds(d: bytes, p: Parse = None, variant: int = 2, tune=TUNE):
    """The kernel's rounds and probes-tried-alone for one block, in order: (list of Round, list of Probe)."""
    if p is None:
        p = parse(d)
    n = len(d)
    shift = shift_of(n)
    mflimit = n - 12
    _, probe_max, wide_min = tune
    rs, pf = [], []
    for li, lp in enumerate(p.loops):
        if lp.after < 0:
            org, A0, fused, wide = -2, 67, False, False
        elif lp.L < probe_max:
            pf.append(Probe(li, lp.m, lp.post_hit))
            if lp.post_hit:
                continue
            org, A0, fused, wide = lp.m + 1 - 3, 67, False, False
        else:
            org, A0, fused, wide = lp.m - 2, 65, True, lp.L >= wide_min
        # the serial probes are where the kernel's formula puts them
        for a, pos in lp.probes:
            assert position(lp.m + 1 - 3 if lp.after >= 0 else -2, a) == pos
        e = lp.end_attempt - A0                   # the loop's event, as an iteration index from A0
        k, A = 0, A0
        while True:
            W = 2 if wide and variant == 2 else 1
            c = 32 * W
            simple = A + c - 1 <= 128 and org + A - 64 + c + 1 <= mflimit
            pos, valid, hs = [], [], []
            for i in range(c):
                a = A + i
                special = fused and k == 0 and i < 2
                x = position(org, a) - (1 if special and i == 0 else 0)
                ok = special or x + (a >> 6) <= mflimit
                pos.append(x); valid.append(ok)
                hs.append(hash_of(int.from_bytes(d[x:x + 4], "little"), shift) if ok else None)
            assert all(valid[:sum(valid)]), "valid iterations are a prefix"
            f = e - (A - A0) if e < A - A0 + c else c
            event = "" if f == c else ("finish" if lp.end == "finish" else "hit")
            if event == "finish":
                assert f == sum(valid)
            by = {}
            for i, hv in enumerate(hs):
                if hv is not None:
                    by.setdefault(hv, []).append(i)
            groups = sorted(g for g in by.values() if len(g) > 1)
            big = max((len(g) for g in groups), default=0)
            path = "exact" if variant == 1 or big >= 3 else ("pair" if big == 2 else "none")
            rs.append(Round(li, k, A, W, fused and k == 0, simple, org, pos, valid, hs, groups, f, event, path))
            if f < c:
                break
            A += c; k += 1; wide = True
    return rs, pf


def counts(d: bytes, variant: int = 2, tune=TUNE) -> dict:
    """The kernel's event counters (enc_prof.cuh) for one block, from the model."""
    p = parse(d)
    rs, pf = rounds(d, p, variant, tune)
    return {"blocks": 1, "seqs": len(p.seqs) + 1, "rounds": len(rs), "rounds_wide": sum(r.W == 2 for r in rs),
            "exact": sum(r.path == "exact" for r in rs), "pair": sum(r.path == "pair" for r in rs),
            "probes": len(pf), "probe_hits": sum(q.hit for q in pf)}


def noise(n: int, seed: int) -> np.ndarray:
    return np.random.default_rng([seed, n]).integers(0, 256, n, dtype=np.uint8)


# ---------------------------------------------------------------------------------------------------------------------
# Constructed blocks: noise (no accidental matches) with words planted at chosen iterations of chosen rounds.  Every
# builder asserts through the model, under variant 2 and the default tune, that the structure it planted is there: the
# round, the sharer group, f and the hit or miss it expects.  A builder that cannot get its structure from a few seeds
# raises, so a change of the kernel's rounds that moves a case fails instead of testing something else.

class Missed(Exception):
    """This seed did not give the planted structure (an accidental hash collision): try the next one."""


def want(cond, what=""):
    if not cond:
        raise Missed(what)


class Block:
    def __init__(self, n: int, seed: int, base=None):
        self.d = noise(n, seed) if base is None else base.copy()
        self.n, self.shift = n, shift_of(n)
        self.rng = np.random.default_rng([seed, n, 99])

    def bytes(self) -> bytes:
        return self.d.tobytes()

    def model(self, variant=2, tune=TUNE):
        b = self.bytes()
        p = parse(b)
        rs, pf = rounds(b, p, variant, tune)
        return p, rs, pf

    def round(self, loop: int, k: int) -> Round:
        _, rs, _ = self.model()
        r = [r for r in rs if r.loop == loop and r.k == k]
        want(r, f"no round {k} in loop {loop}")
        return r[0]

    def word(self, pos: int) -> int:
        return int.from_bytes(self.d[pos:pos + 4].tobytes(), "little")

    def put(self, pos: int, w: int):
        self.d[pos:pos + 4] = np.frombuffer(w.to_bytes(4, "little"), np.uint8)

    def copy(self, src: int, dst: int, length: int = 4):
        for i in range(length):                           # forward, byte by byte: overlapping copies repeat a period
            self.d[dst + i] = self.d[src + i]

    def words(self, k: int, bucket=None) -> list:
        """k distinct words with one hash (a random bucket unless given)."""
        if bucket is None:
            bucket = int(self.rng.integers(0, 1 << (32 - self.shift)))
        out = []
        while len(out) < k:
            w = word_with_hash(bucket, self.shift, int(self.rng.integers(0, 1 << self.shift)))
            if w not in out:
                out.append(w)
        return out

    def match(self, i_pos: int, j_pos: int, length: int) -> int:
        """A match found at j_pos with source i_pos, `length` bytes long: returns its end."""
        self.copy(i_pos, j_pos, length)
        m = j_pos + length
        if self.d[m] == self.d[i_pos + length]:
            self.d[m] ^= 0x5A
        return m

    def collide_tail(self, m: int):
        """Sets the bytes m+2, m+3 so that the words at m-2 and m share a hash but differ."""
        b0 = self.d[m - 2:m + 2].astype(np.uint32)
        lo = np.arange(1 << 16, dtype=np.uint64)
        w2 = np.uint64(int(b0[0]) | int(b0[1]) << 8 | int(b0[2]) << 16 | int(b0[3]) << 24)
        w = np.uint64(int(self.d[m]) | int(self.d[m + 1]) << 8) | (lo << np.uint64(16))
        h = ((w * np.uint64(MULT)) & np.uint64(0xFFFFFFFF)) >> np.uint64(self.shift)
        h2 = ((w2 * np.uint64(MULT)) & np.uint64(0xFFFFFFFF)) >> np.uint64(self.shift)
        ok = np.nonzero((h == h2) & (w != w2))[0]
        want(len(ok), "no colliding tail")
        v = int(ok[0])
        self.d[m + 2], self.d[m + 3] = v & 0xFF, v >> 8


def found(p: Parse, pos: int):
    """Offset of the sequence the serial parse finds at pos, or None."""
    for _, f, ip, ref, _ in p.seqs:
        if f == pos:
            return ip - ref
    return None


@dataclass
class Case:
    name: str
    data: bytes
    facts: dict


def build(name: str, fn, seed: int, tries: int = 40) -> Case:
    for s in range(seed, seed + tries):
        try:
            data, facts = fn(s)
            return Case(name, data, facts)
        except Missed:
            continue
    raise AssertionError(f"{name}: no seed gave the planted structure")


def check_round(r: Round, group=None, f=None, path=None, event=None, simple=None, W=None):
    if group is not None:
        want(sorted(group) in r.groups, f"group {group} not in {r.groups}")
    if f is not None:
        want(r.f == f, f"f {r.f} != {f}")
    if path is not None:
        want(r.path == path, f"path {r.path} != {path}")
    if event is not None:
        want(r.event == event)
    if simple is not None:
        assert r.simple == simple, "the round's form moved"
    if W is not None:
        assert r.W == W, "the round's width moved"


# ---- the catalogue ----------------------------------------------------------------------------------------------------
# Loop 0 of a noise block is the block start's find-match loop: round 0 = attempts 67..98 (32 wide, SIMPLE, positions
# 1..32), round 1 = attempts 99..162 (64 wide, step 1 up to attempt 128 = iteration 29, then 2), rounds 4 and 5 step 4-6.

def _pair(n, k, i, j, simple, W):
    """Iterations i < j of round k of the block start's loop hold one word: j hits with i as its candidate."""
    def fn(s):
        b = Block(n, s)
        r = b.round(0, k)
        b.put(r.pos[i], b.words(1)[0])
        b.copy(r.pos[i], r.pos[j])
        p, _, _ = b.model()
        r = b.round(0, k)
        check_round(r, [i, j], f=j, path="pair", event="hit", simple=simple, W=W)
        want(found(p, r.pos[j]) == r.pos[j] - r.pos[i])
        return b.bytes(), {"round": (0, k), "group": [i, j], "f": j}
    return fn


def _after_match(b, wide):
    """A first match with a literal run of 60 (the fused round after it is 64 wide) or 15 (32 wide).  Returns its end m."""
    r = b.round(0, 1 if wide else 0)
    i, j = (20, 27) if wide else (8, 14)
    b.put(r.pos[i], b.words(1)[0])
    return b.match(r.pos[i], r.pos[j], 8), r.pos[i] + 8


def _fused_pair(i, j, wide):
    """Iterations i < j of the fused round after a match hold one word; i = 0 is the insert of ip-2, i = 1 the probe of ip."""
    def fn(s):
        b = Block(2000, s)
        m, _ = _after_match(b, wide)
        r = b.round(1, 0)
        if i >= 2:
            b.put(r.pos[i], b.words(1)[0])
        b.copy(r.pos[i], r.pos[j])
        p, _, _ = b.model()
        r = b.round(1, 0)
        assert r.fused and r.pos[:2] == [m - 2, m]
        check_round(r, [i, j], f=j, path="pair", event="hit", simple=True, W=2 if wide else 1)
        want(found(p, r.pos[j]) == r.pos[j] - r.pos[i])
        return b.bytes(), {"round": (1, 0), "group": [i, j], "f": j}
    return fn


def _two_words(k, x_idx, i, j, hits):
    """One bucket: an older position x (round 0) and iterations i < j of round k.  hits=False: x and j hold A, i holds B
    (j's candidate is i: a miss).  hits=True: x holds B, i and j hold A (j hits i)."""
    def fn(s):
        b = Block(4000, s)
        x = b.round(0, 0).pos[x_idx]
        r = b.round(0, k)
        A, B = b.words(2)
        b.put(x, B if hits else A); b.put(r.pos[i], A if hits else B); b.put(r.pos[j], A)
        p, _, _ = b.model()
        r = b.round(0, k)
        check_round(r, [i, j], path="pair")
        want(p.refs.get(r.pos[i]) == x)
        want(found(p, r.pos[j]) == (r.pos[j] - r.pos[i] if hits else None))
        return b.bytes(), {"round": (0, k), "group": [i, j], "x": x}
    return fn


def _final_value(f_idx, group, words, who):
    """Round 4 of the block start's loop (64 wide, step 4-5) ends with a hit at f_idx (a copy of a word of round 0, or the
    word of the group's first iteration when f_idx is in the group); the group's iterations hold `words` (letters, one
    bucket); x (round 0) holds A.  A probe of the fused round after the match holds A and shows the bucket's final value:
    `who` = 'x' (no sharer ran), or the index of the last sharer that ran."""
    def fn(s):
        b = Block(4000, s)
        r0 = b.round(0, 0)
        x, y = r0.pos[4], r0.pos[20]
        r = b.round(0, 4)
        ws = dict(zip("ABC", b.words(3)))
        if f_idx in group:
            ws["A"] = b.word(y)
            ws["B"], ws["C"] = [w for w in b.words(3, hash_of(ws["A"], b.shift)) if w != ws["A"]][:2]
        else:
            b.put(x, ws["A"])
            b.copy(y, r.pos[f_idx])
        for g, w in zip(group, words):
            b.put(r.pos[g], ws[w])
        p, _, _ = b.model()
        r = b.round(0, 4)
        check_round(r, group, f=f_idx, path="pair" if len(group) == 2 else "exact", event="hit", simple=False, W=2)
        z = b.round(1, 0).pos[10]
        b.put(z, ws["A"])
        p, _, _ = b.model()
        want(b.round(0, 4).groups == r.groups)
        src = x if who == "x" else r.pos[who]
        want(found(p, z) == z - src, "the bucket's final value does not show")
        return b.bytes(), {"round": (0, 4), "group": group, "f": f_idx, "final": src}
    return fn


def _exact(n, k, group, words, hit_j=None, z_round=None):
    """Three or more iterations of round k of the block start's loop in one bucket with the given letters (the exact
    path).  hit_j: the sharer that hits (the latest earlier sharer holds its word), else none hits.  z_round: (loop,
    round, index) of a later probe holding the word of the last sharer that ran, which must find that sharer."""
    def fn(s):
        b = Block(n, s)
        r = b.round(0, k)
        letters = sorted(set(words))
        ws = dict(zip(letters, b.words(len(letters))))
        for g, w in zip(group, words):
            b.put(r.pos[g], ws[w])
        p, _, _ = b.model()
        r = b.round(0, k)
        check_round(r, group, path="exact")
        if hit_j is not None:
            prev = max(g for g in group if g < hit_j and words[group.index(g)] == words[group.index(hit_j)])
            want(r.f == hit_j and found(p, r.pos[hit_j]) == r.pos[hit_j] - r.pos[prev])
        else:
            want(r.f > max(group) and all(found(p, r.pos[g]) is None for g in group))
        if z_round is not None:
            last = r.pos[max(g for g in group if g <= r.f)]  # the last sharer that ran
            z = b.round(*z_round[:2]).pos[z_round[2]]
            b.copy(last, z)
            p, _, _ = b.model()
            want(b.round(0, k).groups == r.groups and found(p, z) == z - last)
        return b.bytes(), {"round": (0, k), "group": group}
    return fn


def _lanes01(equal, wide):
    """The fused round's lanes 0 and 1 (ip-2 and ip) in one bucket.  equal: one word, lane 1 hits ip-2 (offset 2, no
    literals); else two words, and an older position holds ip's word (lane 1 must still miss: its candidate is ip-2)."""
    def fn(s):
        b = Block(2000, s)
        m, src_end = _after_match(b, wide)
        if equal:
            b.d[m:m + 4] = np.concatenate([b.d[m - 2:m]] * 2)
        else:
            b.collide_tail(m)
        want(b.d[m] != b.d[src_end])
        if not equal:
            b.put(b.round(0, 0).pos[24 if wide else 2], b.word(m))
        p, _, _ = b.model()
        r = b.round(1, 0)
        check_round(r, [0, 1], W=2 if wide else 1)
        want(r.fused and (r.f == 1) == equal and found(p, m) == (2 if equal else None))
        return b.bytes(), {"round": (1, 0), "group": [0, 1], "f": r.f}
    return fn


def _probe_first(equal):
    """A match with 6 literals: the post-match probe is tried alone (default probe_max 8) and ip-2, ip share a bucket
    (h == h2): one word (hit at offset 2) or two."""
    def fn(s):
        b = Block(2000, s)
        r = b.round(0, 0)
        m = b.match(r.pos[1], r.pos[5], 8)
        if equal:
            b.d[m:m + 4] = np.concatenate([b.d[m - 2:m]] * 2)
        else:
            b.collide_tail(m)
        want(b.d[m] != b.d[r.pos[1] + 8])
        p, rs, pf = b.model()
        want(found(p, r.pos[5]) == 4 and len(pf) >= 1 and pf[0].m == m and pf[0].hit == equal)
        want(hash_of(b.word(m), b.shift) == hash_of(b.word(m - 2), b.shift))
        want(found(p, m) == (2 if equal else None))
        return b.bytes(), {"probe": m, "hit": equal}
    return fn


def _far(kind, D):
    """General variant (70 000 bytes, 12-bit hash, u32 table): the table's candidate for a probe at y lies exactly D
    (65 535: a hit, 65 536: a miss) back, at a position x of the block start's first round, whose bucket no other probe
    touched.  A match near 66 KiB makes the loop after it probe consecutive positions; y is
      'pair':  iteration 10 of the fused round after it, sharing its bucket with iteration 30 (another word);
      'exact': the same with iterations 30 and 40;
      'fused': the fused round's lane 1 (y = the match end);
      'probe': the end of a zero-literal match (offset 2) that follows, so the probe at y is tried alone."""
    def fn(s):
        b = Block(70000, s)
        x = 30
        y = x + D
        m = y - 9 if kind in ("pair", "exact") else (y - 4 if kind == "probe" else y)
        p0 = parse(b.bytes())
        pr = [q for q in p0.probes if q <= m - 8]
        j, i = pr[-1], pr[-2]
        b.match(i, j, m - j)
        if kind == "probe":                                 # the zero-literal match m .. y
            b.d[m:m + 4] = np.concatenate([b.d[m - 2:m]] * 2)
            want(b.d[m] != b.d[i + m - j])
        used = set()
        for q in parse(b.bytes()).probes:
            if x - 3 <= q <= y + 3:
                used.add(hash_of(b.word(q), b.shift))
        free = [h for h in range(1 << (32 - b.shift)) if h not in used]
        bucket = free[int(b.rng.integers(0, len(free)))]
        A, B, C = b.words(3, bucket)
        b.put(x, A); b.put(y, A)
        if kind == "probe":
            want(b.d[y] != b.d[m - 2] and b.d[y + 4] != b.d[m + 2])
        p, rs, pf = b.model()
        if kind in ("pair", "exact"):
            r = b.round(1, 0)
            assert r.fused and r.pos[10] == y
            b.put(r.pos[30], B)
            if kind == "exact":
                b.put(r.pos[40], C)
            p, rs, pf = b.model()
            check_round(b.round(1, 0), [10, 30] if kind == "pair" else [10, 30, 40], path=kind)
        elif kind == "fused":
            r = b.round(1, 0)
            want(r.fused and r.pos[1] == y and r.f == (1 if D == 65535 else r.f))
        else:
            want(found(p, m) == 2 and any(q.m == y and q.hit == (D == 65535) for q in pf))
        want(p.refs.get(y) == x, "x is not the candidate at y")
        want(found(p, y) == (D if D == 65535 else None))
        return b.bytes(), {"x": x, "y": y}
    return fn


def _boundary(n):
    """The same planted pattern in the last full round of the block start's loop of a 65 547-byte noise block, at n =
    65 547 (general variant) and cut to 65 546 (64 K variant): A,B,A at iterations 1, 5, 9 (one 13-bit bucket, so one
    12-bit bucket too) and a pair hit at 12, 15."""
    def fn(s):
        full = Block(65547, s)
        _, rs, _ = full.model()
        k = max(r.k for r in rs if r.loop == 0) - 1
        r = full.round(0, k)
        A, B = Block(65546, s).words(2)                    # (one 13-bit hash)
        full.put(r.pos[1], A); full.put(r.pos[5], B); full.put(r.pos[9], A)
        full.put(r.pos[12], full.words(1)[0]); full.copy(r.pos[12], r.pos[15])
        b = full if n == 65547 else Block(n, s, full.d[:n])
        p, _, _ = b.model()
        rr = b.round(0, k)
        check_round(rr, [1, 5, 9], f=15, path="exact", event="hit")
        want(found(p, r.pos[15]) == r.pos[15] - r.pos[12] and found(p, r.pos[9]) is None)
        return b.bytes(), {"round": (0, k)}
    return fn


def catalogue():
    """Every constructed block, as a list of Case."""
    cs = []
    for t in range(1, 32):
        cs.append(build(f"pair-distance-{t}", _pair_dist(t), seed=100 + t))
    for i, j in ((0, 31), (0, 32), (0, 63), (31, 32), (31, 63), (32, 63), (28, 29), (29, 30)):
        cs.append(build(f"pair-wide-{i}-{j}", _pair(4000, 1, i, j, False, 2), seed=200 + i + j))
    for k, i, j in ((2, 3, 40), (2, 40, 50), (5, 10, 60)):
        cs.append(build(f"pair-step-r{k}-{i}-{j}", _pair(4000, k, i, j, False, 2), seed=300 + i + j))
    for i, j, wide in ((2, 32, True), (31, 32, True), (2, 63, True), (31, 63, True), (33, 62, True), (0, 5, True),
                       (0, 40, True), (1, 20, True), (0, 10, False), (1, 3, False), (2, 31, False)):
        cs.append(build(f"pair-fused-{'w' if wide else 'n'}-{i}-{j}", _fused_pair(i, j, wide), seed=400 + i + j))
    for i, j in ((3, 40), (33, 60)):
        for hits in (False, True):
            cs.append(build(f"two-words-{i}-{j}-{'hit' if hits else 'miss'}", _two_words(1, 5, i, j, hits), seed=500 + i))
    cs.append(build("final-none-ran", _final_value(2, [22, 45], "BC", "x"), seed=600))
    cs.append(build("final-earlier-hits", _final_value(2, [2, 25], "AB", 2), seed=610))
    cs.append(build("final-between", _final_value(6, [2, 30], "AA", 2), seed=620))
    cs.append(build("exact-ABA-r0", _exact(4000, 0, [3, 12, 22], "ABA"), seed=700))
    cs.append(build("exact-ABA-half1", _exact(4000, 1, [33, 40, 50], "ABA"), seed=710))
    cs.append(build("exact-ABA-cross", _exact(4000, 1, [5, 30, 40], "ABA"), seed=720))
    cs.append(build("exact-ABB-cross", _exact(4000, 1, [20, 25, 45], "ABB", hit_j=45), seed=730))
    cs.append(build("exact-AABA-middle", _exact(4000, 4, [2, 8, 30, 45], "AABA", hit_j=8, z_round=(1, 0, 10)), seed=740))
    cs.append(build("exact-ABB-r0", _exact(600, 0, [4, 11, 20], "ABB", hit_j=20), seed=745))
    cs.append(build("exact-distinct-4", _exact(4000, 0, [1, 9, 17, 25], "ABCD"), seed=750))
    cs.append(build("exact-distinct-64", _exact(4000, 5, list(range(64)), [chr(0x100 + g) for g in range(64)],
                                                z_round=(0, 6, 5)), seed=760))
    for equal in (True, False):
        for wide in (False, True):
            cs.append(build(f"lanes01-{'equal' if equal else 'distinct'}-{'w' if wide else 'n'}", _lanes01(equal, wide),
                            seed=800 + 2 * equal + wide))
        cs.append(build(f"probe-first-{'hit' if equal else 'miss'}", _probe_first(equal), seed=850 + equal))
    for kind in ("pair", "exact", "fused", "probe"):
        for D in (65535, 65536):
            cs.append(build(f"far-{kind}-{D}", _far(kind, D), seed=900 + D % 2))
    for n in (65546, 65547):
        cs.append(build(f"boundary-{n}", _boundary(n), seed=1000))
    return cs


def _pair_dist(t):
    """Iterations i and i + t of the block start's first round (32 wide, SIMPLE) hold one word: the later one hits at lane
    distance t (t < 4: the words overlap, a run with period t)."""
    i = (5 * t) % (32 - t)
    return _pair(600, 0, i, i + t, True, 1)
