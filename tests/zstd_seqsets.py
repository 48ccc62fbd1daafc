"""Test support: hand-built inputs for stage E of the Zstandard encoder (the entropy coder, csrc/zstd_enc_entropy.cu).

Stage E codes whatever sequences and literals the parse hands it.  The sets here are built in plain Python so that they reach the
branches of stage E that real parses rarely or never reach: every literals form and header size, deep Huffman trees, both Huffman
descriptions, every sequence-count form, each table mode per symbol type, every literal-length and match-length code, offset codes
up to 27, the RLE block and its near misses, the raw fallbacks, and groups of blocks of very different kinds side by side.

A `Case` is a frame log and a list of blocks; a block is a list of (litLength, matchLength, offBase) and its literal bytes.  `build`
executes the sequences (repcodes as RFC 8878 3.1.1.5 resolves them, history {1, 4, 8} at each frame start, carried across the
frame's blocks) into the input `src`, in the dense layout of the oracle's b2zo_zstd_find_sequences.  Every block but the last is
131 072 bytes, so the encoder cuts the input into exactly these blocks and frames.  A case marked `parity_only` has offsets that
reach before its frame start (offset codes up to 27 in small frames): its blocks are compared byte for byte, never decoded.

Every case names the branch it is built for and states it in `expect` (block index -> fields of `read_block`), so that a change to
stage E's decisions fails the case that targets it instead of passing as one more round trip.
"""
import heapq
import random
import struct

import numpy as np

import zstd_craft as C

BLOCK = 131072
MAXSEQ = 32768


class Case:
    def __init__(self, name, frame_log=17, parity_only=False):
        self.name, self.frame_log, self.parity_only = name, frame_log, parity_only
        self.blocks = []                                        # [(seqs [(ll, ml, offBase)], literal bytes)]
        self.expect = {}                                        # block index -> {read_block field: value or predicate}
        self.src = None

    def add(self, seqs, lits, **expect):
        if expect:
            self.expect[len(self.blocks)] = expect
        self.blocks.append((list(seqs), bytes(lits)))
        return self

    # ---- execution
    def build(self):
        if self.src is not None:
            return self
        F = 1 << self.frame_log
        out = bytearray()
        f0, reps = 0, None
        for b, (seqs, lits) in enumerate(self.blocks):
            assert len(seqs) <= MAXSEQ, (self.name, b)
            if len(out) % F == 0:
                f0, reps = len(out), [1, 4, 8]
            start, lp = len(out), 0
            for ll, ml, ob in seqs:
                assert ml >= 3 and 0 < ob < (1 << 28) and ll < (1 << 18) and ml < (1 << 18), (self.name, b, ll, ml, ob)
                out += lits[lp:lp + ll]; lp += ll
                off, reps = C.resolve_offset(reps, ob, ll)
                if not 0 < off <= len(out) - f0:
                    assert self.parity_only, (self.name, b, off, len(out) - f0)
                    out += bytes(ml)                            # nothing to copy from: the bytes of a set that is never decoded
                    continue
                s = len(out) - off
                if off >= ml:
                    out += out[s:s + ml]
                else:
                    out += (out[s:] * (ml // off + 1))[:ml]
            assert lp <= len(lits), (self.name, b)
            out += lits[lp:]
            size = len(out) - start
            assert size == BLOCK or (b == len(self.blocks) - 1 and 0 < size <= BLOCK), (self.name, b, size)
        self.src = bytes(out)
        return self

    @property
    def n(self):
        return len(self.build().src)

    def frames(self):
        """[(first block, block count, frame bytes)]"""
        F, n = 1 << self.frame_log, self.n
        return [(f0 // BLOCK, (min(F, n - f0) + BLOCK - 1) // BLOCK, min(F, n - f0)) for f0 in range(0, n, F)]

    def last_flags(self):
        flags = [0] * len(self.blocks)
        for b0, nb, _ in self.frames():
            flags[b0 + nb - 1] = 1
        return flags

    def arrays(self):
        """(src, seqs, nseq, lits, nlit) in the oracle's dense block layout, with the padding the kernels' word loads may touch"""
        self.build()
        nb = len(self.blocks)
        seqs = np.zeros(nb * MAXSEQ, dtype=np.uint64); nseq = np.zeros(nb, dtype=np.uint32)
        lits = np.zeros(nb * BLOCK + 64, dtype=np.uint8); nlit = np.zeros(nb, dtype=np.uint32)
        for b, (sq, lt) in enumerate(self.blocks):
            if sq:
                a = np.array(sq, dtype=np.uint64)
                seqs[b * MAXSEQ:b * MAXSEQ + len(sq)] = a[:, 2] | (a[:, 0] << np.uint64(28)) | (a[:, 1] << np.uint64(46))   # B2Z_PACK_SEQ
            nseq[b] = len(sq)
            lits[b * BLOCK:b * BLOCK + len(lt)] = np.frombuffer(lt, dtype=np.uint8); nlit[b] = len(lt)
        src = np.zeros(self.n + 64, dtype=np.uint8); src[:self.n] = np.frombuffer(self.src, dtype=np.uint8)
        return src, seqs, nseq, lits, nlit


# ---------------------------------------------------------------- frames around the blocks
def frame_header(n, window_log):
    """the encoder's frame header (zstd_enc_oracle.c write_frame_header): 4-byte content size, the smallest window >= the frame"""
    wl = 10
    while (1 << wl) < n and (wl < window_log or wl < 17):
        wl += 1
    return struct.pack("<IBBI", C.MAGIC, 0x80, (wl - 10) << 3, n)


def assemble(case, blocks):
    """the coded blocks (list of bytes, one per block) as the encoder's frames, without size hints"""
    out = bytearray()
    for b0, nb, fn in case.frames():
        out += frame_header(fn, case.frame_log) + b"".join(blocks[b0:b0 + nb])
    return bytes(out)


def split_blocks(data, sizes):
    out, p = [], 0
    for s in sizes:
        out.append(bytes(data[p:p + int(s)])); p += int(s)
    return out


# ---------------------------------------------------------------- reading a coded block back
def _read_ncount(buf, pos, max_sym):
    """FSE table description at buf[pos:] (RFC 8878 4.1.1) -> (accuracy log, bytes)"""
    bits = int.from_bytes(bytes(buf[pos:pos + 80]), "little")
    p = 0

    def take(n):
        nonlocal p
        v = (bits >> p) & ((1 << n) - 1); p += n; return v
    log = take(4) + 5
    remaining, s = 1 << log, 0
    while remaining > 0 and s <= max_sym:
        nb = (remaining + 1).bit_length()
        T = 1 << (nb - 1); mx = 2 * T - 1 - (remaining + 1)
        v = (bits >> p) & ((1 << (nb - 1)) - 1)
        if v < mx:
            p += nb - 1
        else:
            v = take(nb)
            if v >= T:
                v -= mx
        proba = v - 1
        remaining -= 1 if proba < 0 else proba
        s += 1
        if proba == 0:
            while True:
                r = take(2); s += r
                if r < 3:
                    break
    assert remaining == 0, "bad table description"
    return log, (p + 7) // 8


def read_block(blk):
    """the decisions visible in one coded block: block type and size; literals type, header bytes, count, stream count and Huffman
    description (form, its FSE log); sequence count and its header form; the three table modes and logs"""
    h = int.from_bytes(blk[:3], "little")
    r = dict(last=h & 1, btype=("raw", "rle", "compressed")[(h >> 1) & 3], size=h >> 3)
    if r["btype"] != "compressed":
        return r
    body = blk[3:3 + r["size"]]
    b0 = body[0]; lt = b0 & 3; sf = (b0 >> 2) & 3
    r["lit"] = ("raw", "rle", "huf", "treeless")[lt]
    if lt <= 1:
        lh = 1 if sf in (0, 2) else (2 if sf == 1 else 3)
        v = int.from_bytes(body[:lh], "little")
        r["nlit"] = v >> 3 if lh == 1 else v >> 4
        sec = lh + (r["nlit"] if lt == 0 else 1)
        r["streams"] = 1
    else:
        lh = 3 if sf <= 1 else sf + 2
        v = int.from_bytes(body[:lh], "little")
        w = {3: 10, 4: 14, 5: 18}[lh]
        r["nlit"] = (v >> 4) & ((1 << w) - 1); csize = v >> (4 + w)
        r["streams"] = 1 if sf == 0 else 4
        sec = lh + csize
        d = body[lh]
        r["huf_desc"] = "fse" if d < 128 else "direct"
        if d < 128:
            r["huf_log"] = (body[lh + 1] & 15) + 5
        else:
            r["huf_nw"] = d - 127
    r["lit_hdr"] = lh
    p = sec
    c0 = body[p]
    if c0 < 128:
        r["nbseq"], r["seq_form"], p = c0, 1, p + 1
    elif c0 < 255:
        r["nbseq"], r["seq_form"], p = ((c0 - 128) << 8) + body[p + 1], 2, p + 2
    else:
        r["nbseq"], r["seq_form"], p = body[p + 1] + (body[p + 2] << 8) + 0x7F00, 3, p + 3
    if r["nbseq"]:
        m = body[p]; p += 1
        modes, logs = [], []
        for k, (sh, dlog, mx) in zip(("ll", "of", "ml"), ((6, 6, 35), (4, 5, 31), (2, 6, 52))):
            mode = ("pre", "rle", "fse", "rep")[(m >> sh) & 3]
            modes.append(mode)
            if mode == "pre":
                logs.append(dlog)
            elif mode == "rle":
                logs.append(0); p += 1
            else:
                lg, nbytes = _read_ncount(body, p, mx); logs.append(lg); p += nbytes
        r["modes"], r["logs"] = tuple(modes), tuple(logs)
    return r


def check_branches(case, blocks):
    """every block's Last_Block flag, and the fields the case expects"""
    for b, (blk, last) in enumerate(zip(blocks, case.last_flags())):
        assert blk[0] & 1 == last, (case.name, b)
    for b, want in case.expect.items():
        got = read_block(blocks[b])
        for k, v in want.items():
            ok = v(got.get(k)) if callable(v) else got.get(k) == v
            assert ok, (case.name, b, k, got.get(k), v, got)


# ---------------------------------------------------------------- building blocks
def skewed(rng, n, alphabet):
    a = np.asarray(list(alphabet), dtype=np.uint8)
    p = 1.0 / np.arange(1, len(a) + 1) ** 1.3
    return bytes(rng.choice(a, size=n, p=p / p.sum()).tolist())


def noise(rng, n):
    return rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()


def lit_block(lits, size=BLOCK):
    """a block of `size` bytes whose literals are `lits`, the rest one match on the literals (two when there is one literal: one
    literal and a match of offset 1 over the whole block is the RLE block)"""
    n = len(lits)
    assert 1 <= n and size - n >= 3
    if n == 1:
        return [(1, 3, 4), (0, size - 4, 4)], lits
    return [(n, size - n, 2 + 3)], lits


def rle_block(byte=0, size=BLOCK):
    """the single sequence the parse emits for a block of one repeated byte"""
    return [(1, size - 1, 4)], bytes([byte])


def seq_block(rng, nseq, frame_pos, size=BLOCK, ll_max=2, ml_extra=None, off_max=1 << 16, rep=0.3, lit_alpha=range(16),
              ll0=0.3, fixed_ll=None, fixed_ml=None, off_range=None):
    """nseq valid sequences filling a block of `size` bytes that starts frame_pos bytes into its frame; returns (seqs, lits, the
    repcode history after them).  ml_extra: bytes spread over the match lengths beyond 3 each (default: whatever
    the block has left over after the literals, which then end the block as trailing literals when ml_extra is given)"""
    rnd = random.Random(int(rng.integers(1 << 30)))
    lls = [fixed_ll if fixed_ll is not None else (0 if rnd.random() < ll0 else rnd.randint(1, ll_max)) for _ in range(nseq)]
    if frame_pos == 0 and lls and lls[0] == 0:
        lls[0] = 1
    mls = [fixed_ml if fixed_ml is not None else 3 for _ in range(nseq)]
    room = size - sum(lls) - sum(mls)
    while room < 0:                                                 # too many literals for the block: drop some
        i = rnd.randrange(1 if frame_pos == 0 else 0, nseq)
        if lls[i]:
            lls[i] -= 1; room += 1
    if fixed_ml is None:
        extra = room if ml_extra is None else min(ml_extra, room)
        k = 0
        while extra > 0 and nseq:                                   # spread it in random pieces (the last piece may be large)
            i = rnd.randrange(nseq); step = min(extra, rnd.choice((1, 2, 5, 13, 40, 300)) if k < 4 * nseq else extra)
            mls[i] += step; extra -= step; k += 1
    trailing = size - sum(lls) - sum(mls)
    reps = [1, 4, 8]
    seqs, pos, explicit = [], frame_pos, 0
    for ll, ml in zip(lls, mls):
        pos += ll
        ob = None
        # repcodes only once three offsets of this block fill the history, as the parses do: a decoder keeps no history through a
        # block the encoder stores raw, so a repcode may not lean on an earlier block's sequences
        if explicit >= 3 and rnd.random() < rep:
            cand = rnd.randint(1, 3)
            off, _ = C.resolve_offset(reps, cand, ll)
            if 0 < off <= pos:
                ob = cand
        if ob is None:
            if off_range:
                lo, hi = off_range
                off = rnd.randint(lo, min(hi, pos))
            else:
                off = rnd.randint(1, min(pos, off_max))
            assert off >= 1
            ob = off + 3; explicit += 1
        _, reps = C.resolve_offset(reps, ob, ll)
        seqs.append((ll, ml, ob)); pos += ml
    lits = skewed(rng, sum(lls) + trailing, lit_alpha)
    return seqs, lits, reps


def huf_depth(counts):
    """longest code of an unlimited Huffman code for counts {symbol: count} (heapq; ties do not change the deepest leaf here)"""
    h = [(c, 0, s) for s, c in counts.items() if c]
    heapq.heapify(h)
    k = 1 << 20
    while len(h) > 1:
        a = heapq.heappop(h); b = heapq.heappop(h)
        heapq.heappush(h, (a[0] + b[0], max(a[1], b[1]) + 1, k)); k += 1
    return h[0][1]


def halved(counts, k):
    return {s: (c + (1 << k) - 1) >> k for s, c in counts.items()}


def fib_counts(nsym, stride=11):
    f = [1, 1]
    while len(f) < nsym:
        f.append(f[-1] + f[-2])
    return {(s * stride) % 256: c for s, c in enumerate(f[:nsym])}


def lits_of(rng, counts):
    b = bytearray()
    for s, c in counts.items():
        b += bytes([s]) * c
    a = np.frombuffer(bytes(b), dtype=np.uint8).copy(); rng.shuffle(a)
    return a.tobytes()


def entropy_bytes(seqs, lits):
    """a lower bound of a sequences section's stream + Huffman literals, in bytes: the codes' empirical entropy plus the extra bits"""
    def h(vals):
        _, c = np.unique(np.asarray(vals), return_counts=True); p = c / c.sum()
        return float(-(c * np.log2(p)).sum())
    codes = [[C.ll_code(ll) for ll, _, _ in seqs], [C.ml_code(ml) for _, ml, _ in seqs], [C.of_code(ob) for _, _, ob in seqs]]
    extra = sum(C.LL_BITS[C.ll_code(ll)] + C.ML_BITS[C.ml_code(ml)] + C.of_code(ob) for ll, ml, ob in seqs)
    return (sum(h(c) for c in codes) + extra + h(list(lits))) / 8


# ---------------------------------------------------------------- the sets
def _literal_cases(rng):
    out = []
    # no literals: the block copies the one before it
    out.append(Case("lit-raw-0", 18).add(*rle_block(7)).add([(0, BLOCK, 4)], b"", lit="raw", nlit=0, lit_hdr=1))
    for n in range(1, 8):
        out.append(Case(f"lit-raw-{n}").add(*lit_block(bytes(range(40, 40 + n))), lit="raw", nlit=n, lit_hdr=1))
    out.append(Case("lit-raw-7-equal").add(*lit_block(b"q" * 7), lit="raw", nlit=7))          # one symbol, below the RLE minimum
    for n, hdr in ((8, 1), (31, 1), (32, 2), (4095, 2), (4096, 3)):
        out.append(Case(f"lit-rle-{n}").add(*lit_block(b"z" * n), lit="rle", nlit=n, lit_hdr=hdr))
    out.append(Case("lit-raw-63").add(*lit_block(skewed(rng, 63, range(6))), lit="raw", nlit=63))               # below the Huffman minimum
    for n, streams, hdr in ((64, 1, 3), (255, 1, 3), (256, 4, 3), (257, 4, 3), (1023, 4, 3), (1024, 4, 4), (16383, 4, 4), (16384, 4, 5)):
        out.append(Case(f"lit-huf-{n}").add(*lit_block(skewed(rng, n, range(12))), lit="huf", nlit=n, streams=streams, lit_hdr=hdr))
    out.append(Case("lit-huf-whole-block").add([], skewed(rng, BLOCK, range(40)), btype="compressed", lit="huf", nlit=BLOCK, streams=4, lit_hdr=5))
    return out


def _huffman_cases(rng):
    out = []
    a = np.repeat(np.arange(256, dtype=np.uint8), 16); rng.shuffle(a)
    out.append(Case("huf-256-equal-weights-raw").add(*lit_block(a.tobytes()), lit="raw", nlit=4096))          # > 128 weights, all equal
    # 255 equal counts: one code of 7 bits, the rest 8 -- a valid table that cannot beat raw by its own description's size
    out.append(Case("huf-not-smaller-than-raw").add(*lit_block(lits_of(rng, {s: 16 for s in range(255)})), lit="raw", nlit=4080))
    out.append(Case("huf-two-symbols-0-1").add(*lit_block(lits_of(rng, {0: 1000, 1: 3000})), lit="huf", huf_desc="direct", huf_nw=1))
    out.append(Case("huf-two-symbols-0-255").add(*lit_block(lits_of(rng, {0: 3000, 255: 1000})), lit="huf", huf_desc="fse", huf_log=5))
    one, two = fib_counts(14), {(s * 11) % 256: 1 << s for s in range(16)}          # Fibonacci counts; powers of two
    assert huf_depth(one) > 11 and huf_depth(halved(one, 1)) <= 11, (huf_depth(one), huf_depth(halved(one, 1)))
    assert huf_depth(two) > 11 and huf_depth(halved(two, 1)) > 11, (huf_depth(two), huf_depth(halved(two, 1)))
    out.append(Case("huf-deep-one-halving").add(*lit_block(lits_of(rng, one)), lit="huf"))
    out.append(Case("huf-deep-several-halvings").add(*lit_block(lits_of(rng, two)), lit="huf"))
    out.append(Case("huf-direct-description").add(*lit_block(skewed(rng, 3000, range(4))), lit="huf", huf_desc="direct", huf_nw=3))
    out.append(Case("huf-fse-description-log5").add(*lit_block(skewed(rng, 6000, range(40))), lit="huf", huf_desc="fse", huf_log=5))
    expo = bytes(min(255, int(x)) for x in rng.exponential(30, 20000))
    assert max(expo) > 128
    out.append(Case("huf-over-128-weights-fse").add(*lit_block(expo), lit="huf", huf_desc="fse"))
    # The weights' FSE log is clamped to [5, 6] from min(6, highbit(nw - 1) - 2) and lower bounds that never pass 5 (nw <= 255,
    # weights <= 11), so it is 5 for every table: log 6 cannot be reached and is not a case.
    return out


def _sequence_cases(rng):
    out = []
    for ns in (1, 2, 3, 47, 48, 49, 96, 97, 127, 128, 0x7EFF, 0x7F00, MAXSEQ):
        kw = dict(ll_max=1, ll0=0.5) if ns > 20000 else {}
        sq, lt, _ = seq_block(rng, ns, 0, off_max=1 << (4 + ns % 12), **kw) if ns > 1 else (*lit_block(b"12345"), None)
        form = 1 if ns < 128 else (2 if ns < 0x7F00 else 3)
        out.append(Case(f"nbseq-{ns}").add(sq, lt, nbseq=ns, seq_form=form))
    # nbSeq 0 with literals that do not fill the block: a raw block (the block has nothing to copy)
    out.append(Case("nbseq-0-short", 17).add([], skewed(rng, 5000, range(8)), btype="compressed", nbseq=0, seq_form=1))
    # table modes, one type at a time
    sq, lt, _ = seq_block(rng, 300, 0, fixed_ll=5)
    out.append(Case("mode-rle-ll").add(sq, lt, modes=lambda m: m[0] == "rle" and m[2] != "rle"))
    out.append(Case("mode-rle-of", 18).add(*rle_block(3)).add(*seq_block(rng, 300, BLOCK, rep=0, off_range=(61, 124))[:2],       # OF code 6 only
                                                               modes=lambda m: m[1] == "rle" and m[0] != "rle"))
    sq, lt, _ = seq_block(rng, 300, 0, fixed_ml=4, ml_extra=0)
    out.append(Case("mode-rle-ml").add(sq, lt, modes=lambda m: m[2] == "rle" and m[0] != "rle"))
    # one code per type: RLE tables from three sequences on, the predefined ones for one or two (nbSeq <= 2)
    out.append(Case("mode-one-is-predefined").add([(9, 40, 5 + 3)], noise(rng, BLOCK - 40), modes=("pre", "pre", "pre")))
    out.append(Case("mode-two-same-is-predefined").add([(9, 40, 5 + 3), (9, 41, 6 + 3)], noise(rng, BLOCK - 81), modes=("pre", "pre", "pre")))
    out.append(Case("mode-three-same-is-rle").add([(9, 40, 5 + 3)] * 3, noise(rng, BLOCK - 120), modes=("rle", "rle", "rle"), logs=(0, 0, 0)))
    sq, lt, _ = seq_block(rng, 12, 0, ll_max=30, off_max=5000, rep=0.2)
    out.append(Case("mode-predefined").add(sq, skewed(rng, len(lt), range(8)), modes=("pre", "pre", "pre")))
    # compressed tables: the smallest log (5) from about 20 sequences, LL codes 0 and 35 only (the NCount's zero runs of >= 3)
    sq = [(65536 + 100, 3, 4)] + [(0, 3 + (k % 5), 4 + (k % 7)) for k in range(19)]
    used = sum(a + b for a, b, _ in sq)
    out.append(Case("table-log5-ll-zero-runs").add(sq, skewed(rng, 65536 + 100 + BLOCK - used, range(20)),
                                                   modes=lambda m: m[0] == "fse", logs=lambda g: g[0] == 5))
    # the largest logs, 9 / 8 / 9, from 32 768 sequences of varied codes.  (choose_seq_table's `while ((1u << log) < present) log++`
    # cannot fire: 36 or more present codes need nbSeq >= 36, where the log is already at least 6.)
    sq, lt, _ = seq_block(rng, 20000, 0, ll_max=2, ll0=0.4, off_max=1 << 16)
    out.append(Case("table-largest-logs").add(sq, lt, modes=("fse", "fse", "fse"), logs=(9, 8, 9)))
    # every LL code and every ML code (two blocks each: the largest codes take half a block)
    c = Case("ll-every-code", 18)
    s0 = [(C.LL_BASE[k], 3, 4) for k in (1, 0, *range(2, 35))]                   # offset 1 throughout
    used = sum(a + b for a, b, _ in s0)
    s0.append((0, BLOCK - used, 4))
    c.add(s0, skewed(rng, sum(a for a, _, _ in s0), range(30)), nbseq=36)
    c.add([(65536, BLOCK - 65536, BLOCK + 3)], skewed(rng, 65536, range(30)))
    assert {C.ll_code(a) for b in c.blocks for a, _, _ in b[0]} == set(range(36))
    out.append(c)
    c = Case("ml-every-code", 18)
    s0 = [(1, C.ML_BASE[k], 4 + (k % 3)) for k in range(52)]
    s0[0] = (3, 3, 4)
    used = sum(a + b for a, b, _ in s0)
    c.add(s0, skewed(rng, sum(a for a, _, _ in s0) + BLOCK - used, range(30)), nbseq=52)
    c.add([(1, 65539, 5000), (0, BLOCK - 1 - 65539, 70000)], b"!")
    assert {C.ml_code(b) for blk in c.blocks for _, b, _ in blk[0]} == set(range(53))
    out.append(c)
    # offset codes 0 and 1: real repcodes with litLength 0 and without
    sq, lt, _ = seq_block(rng, 3000, 0, rep=0.6, ll0=0.5, off_max=64)
    obs = {(ob, ll == 0) for ll, _, ob in sq}
    assert all((ob, z) in obs for ob in (1, 2, 3) for z in (False, True))
    out.append(Case("repcodes").add(sq, lt, nbseq=3000, modes=lambda m: m[1] == "fse"))
    return out


def _offset_cases(rng):
    out = []
    # offset codes 0 .. 21 in a valid 4 MiB frame: 31 blocks of one byte each, then sequences reaching back 2^k
    c = Case("offset-codes-to-21", 22)
    for b in range(31):
        c.add(*rle_block(b + 1))
    pos, sq = 31 * BLOCK, []
    for k in range(2, 22):                                          # offBase in [2^k, 2^k + 2^(k-1))
        sq.append((1, 40, (1 << k) + (k * 7919) % (1 << (k - 1)))); pos += 41
    c.add(sq, skewed(rng, BLOCK - 20 * 40, range(10)), nbseq=20)
    assert {C.of_code(ob) for _, _, ob in sq} >= set(range(2, 22))
    out.append(c)
    # offset codes up to 27 (offBase up to 2^28 - 1), reaching before the frame start: compared byte for byte only
    c = Case("offset-codes-to-27-parity", 17, parity_only=True)
    sq = [(1, 30, (1 << k) + (k * 31) % (1 << k)) for k in range(2, 28)]
    c.add(sq, skewed(rng, BLOCK - 26 * 30, range(10)), modes=lambda m: m[1] != "rle")
    assert {C.of_code(ob) for _, _, ob in sq} == set(range(2, 28))
    out.append(c)
    # one sequence of about 85 bits (rare LL 35, ML 51 and OF 27 codes among short ones): its fields pass 64 bits in E3's packing
    sq, lt, _ = seq_block(rng, 8000, 0, ll_max=1, ml_extra=0, off_max=1 << 10)
    wide = (65536, 32771, (1 << 28) - 1)
    used = sum(a + b for a, b, _ in sq)
    rest = BLOCK - used - 65536 - 32771
    out.append(Case("wide-sequence-parity", 17, parity_only=True).add(sq[:4000] + [wide] + sq[4000:], skewed(rng, sum(a for a, _, _ in sq) + 65536 + rest, range(10)),
                                                                      btype="compressed", modes=("fse", "fse", "fse")))
    return out


def _block_cases(rng):
    out = []
    out.append(Case("rle-block").add(*rle_block(9), btype="rle", size=BLOCK))
    out.append(Case("rle-near-miss-offbase-5", 18).add(*rle_block(9)).add([(1, BLOCK - 1, 5)], b"\x09", btype="compressed"))
    out.append(Case("rle-near-miss-ll-2").add([(2, BLOCK - 2, 4)], b"\x09\x09", btype="compressed"))
    out.append(Case("rle-near-miss-1-byte-block").add([], b"\x09", btype="raw", size=1))
    out.append(Case("raw-block-not-smaller").add([], noise(rng, BLOCK), btype="raw", size=BLOCK))
    # over the body cap: 32 768 sequences whose offsets (2^15 .. 2^19) and three compressed tables put the section's upper bound
    # above B2Z_BODY_CAP, while what they would really code to is well under the block: stored raw by the cap alone
    c = Case("body-cap-raw", 20)
    for b in range(7):
        c.add(*rle_block(b + 1))
    sq, _, _ = seq_block(rng, MAXSEQ, 7 * BLOCK, ll_max=2, ll0=0.34, rep=0, off_range=(1 << 15, 1 << 19))
    lt = noise(rng, sum(a for a, _, _ in sq) + BLOCK - sum(a + b for a, b, _ in sq))
    c.add(sq, lt, btype="raw")
    lo = entropy_bytes(sq, lt)
    assert lo < BLOCK - 4096, lo                                    # without the cap the block would be coded
    out.append(c)
    # Last_Block at every frame end and on a ragged final block (checked on every case; here five frames of 256 KiB)
    c = Case("frames-last-flags", 18)
    for b in range(9):
        if b % 3 == 0:
            c.add(*rle_block(b), btype="rle")
        else:
            fp = (b % 2) * BLOCK
            c.add(*seq_block(rng, 40 + 100 * b, fp, off_max=1 << 12)[:2])
    c.add(*seq_block(rng, 50, BLOCK, size=70000, off_max=1 << 12)[:2])
    out.append(c)
    return out


def mixed_case(rng, name, nblk, frame_log=20):
    """nblk blocks of very different kinds side by side: RLE blocks, blocks without sequences, blocks over the body cap (they need
    no FSE chain) beside chained blocks of 1 to 32 768 sequences; the last block ragged when nblk is odd"""
    c = Case(name, frame_log)
    bpf = 1 << (frame_log - 17)
    kinds = ("rle", "seq48", "lits", "seq32768", "seq1", "cap", "seq2000", "seq97", "noise", "seq5")
    for b in range(nblk):
        fp = (b % bpf) * BLOCK
        k = kinds[b % len(kinds)]
        if k == "cap" and (fp < 5 * BLOCK or size < BLOCK):
            k = "seq2000"
        size = BLOCK if b + 1 < nblk or nblk % 2 == 0 else 90001
        if k == "rle":
            c.add(*rle_block(b % 256, size), btype="rle")
        elif k == "lits":
            c.add([], skewed(rng, size, range(20)))
        elif k == "noise":
            c.add([], noise(rng, size), btype="raw")
        elif k == "cap":
            sq, _, _ = seq_block(rng, MAXSEQ, fp, size=size, ll_max=2, ll0=0.34, rep=0, off_range=(1 << 15, 1 << 19))
            c.add(sq, noise(rng, sum(a for a, _, _ in sq) + size - sum(a + b for a, b, _ in sq)), btype="raw")
        else:
            ns = int(k[3:])
            kw = dict(ll_max=1, ll0=0.5) if ns > 20000 else {}
            if fp == 0 and ns == 1:
                c.add(*lit_block(skewed(rng, 500, range(9)), size))
            else:
                c.add(*seq_block(rng, min(ns, size // 4), fp, size=size, off_max=min(fp + 1, 1 << 18) if fp else 1 << 14, **kw)[:2])
    return c


def _grouping_cases(rng):
    return [mixed_case(rng, f"group-{n}-blocks", n) for n in (9, 10, 11, 29, 31)]


_CACHE = None


def cases():
    """every CPU and GPU case, built"""
    global _CACHE
    if _CACHE is None:
        rng = np.random.default_rng(8878)
        out = _literal_cases(rng) + _huffman_cases(rng) + _sequence_cases(rng) + _offset_cases(rng) + _block_cases(rng) + _grouping_cases(rng)
        for c in out:
            c.build()
        names = [c.name for c in out]
        assert len(names) == len(set(names))
        _CACHE = out
    return _CACHE


def one_launch(group):
    """cases of one frame log back to back as one input: every case but the last must end on a frame boundary (a ragged case only
    last), which keeps each block's position in its frame and Last_Block flag"""
    fl = group[0].frame_log
    assert all(c.frame_log == fl for c in group) and all(c.n % (1 << fl) == 0 for c in group[:-1])
    out = Case("+".join(c.name for c in group)[:60] + f"..{len(group)}", fl, parity_only=any(c.parity_only for c in group))
    b = 0
    for c in group:
        for i, blk in enumerate(c.blocks):
            out.blocks.append(blk)
            if i in c.expect:
                out.expect[b + i] = c.expect[i]
        b += len(c.blocks)
    out.src = b"".join(c.src for c in group)
    return out


def launches(group_cases):
    """the cases as few inputs as possible: one per frame log, plus one more for each extra ragged case"""
    by_fl = {}
    for c in group_cases:
        by_fl.setdefault(c.frame_log, []).append(c)
    out = []
    for fl, cs in sorted(by_fl.items()):
        whole = [c for c in cs if c.n % (1 << fl) == 0]
        ragged = [c for c in cs if c.n % (1 << fl)]
        out.append(one_launch(whole + ragged[:1]))
        out += [one_launch([c]) for c in ragged[1:]]
    return out


# ---------------------------------------------------------------- GPU-only sets
def large_offset_case():
    """offset codes up to 26 in a valid 2^27-byte frame: 1 000 RLE blocks, then blocks whose sequences reach back up to 2^27 - 1
    bytes, one of them with a sequence of about 80 bits (LL code 35, ML code 51, OF code 26, rare)"""
    rng = np.random.default_rng(27)
    c = Case("offset-codes-to-26-in-2^27", 27)
    for b in range(1000):
        c.add(*rle_block(b % 251 + 1))
    pos = 1000 * BLOCK
    sq = []
    for k in range(2, 27):
        sq.append((1, 40, (1 << k) + (k * 7919) % (1 << (k - 1)))); pos += 41
    c.add(sq, skewed(rng, BLOCK - 25 * 40, range(10)), modes=lambda m: m[1] != "rle")
    assert {C.of_code(ob) for _, _, ob in sq} >= set(range(2, 27))
    s2, _, _ = seq_block(rng, 8000, pos, ll_max=1, ml_extra=0, off_max=1 << 10)
    wide = (65536, 32771, (1 << 26) + 12345 + 3)
    used = sum(a + b for a, b, _ in s2)
    c.add(s2[:4000] + [wide] + s2[4000:], skewed(rng, sum(a for a, _, _ in s2) + 65536 + BLOCK - used - 65536 - 32771, range(10)), btype="compressed")
    return c.build()


def grid_case(sm_count, ent_warps=4, ctas_per_sm=16):
    """one launch of sm_count * 64 + 37 blocks: stage E's table and bitstream kernels (grid capped at sm_count * 16 CTAs of 4 warps)
    take a second lap of their grid-stride loop for the last 37.  RLE blocks of zeros first, then every full-block case of 128 KiB
    frames, so that the real blocks are the ones that come round on the second lap"""
    real = [c for c in cases() if c.frame_log == 17 and c.n % BLOCK == 0 and len(c.blocks) == 1]
    total = sm_count * ctas_per_sm * ent_warps + 37
    assert len(real) <= total
    pad = Case("zeros", 17)
    for _ in range(total - len(real)):
        pad.add(*rle_block(0))
    return one_launch([pad.build()] + real)


# ---------------------------------------------------------------- the oracle's bytes
def oracle_blocks(case):
    """every block of the case coded by the oracle's compress_block (b2zo_zstd_encode_block): list of bytes"""
    import ctypes
    import helpers
    O = helpers.oracle()
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    O.b2zo_zstd_encode_block.restype = ctypes.c_int64
    O.b2zo_zstd_encode_block.argtypes = [vp, sz, vp, sz, sz, ctypes.c_int, vp, ctypes.c_uint32, vp, ctypes.c_uint32]
    src, seqs, nseq, lits, nlit = case.arrays()
    F, n, last = 1 << case.frame_log, case.n, case.last_flags()
    buf = np.empty(BLOCK + 3, dtype=np.uint8)
    out = []
    for b in range(len(case.blocks)):
        p0 = b * BLOCK; f0 = p0 // F * F
        r = O.b2zo_zstd_encode_block(buf.ctypes.data, buf.size, src.ctypes.data + f0, p0 - f0, min(BLOCK, n - p0), last[b],
                                     seqs.ctypes.data + 8 * b * MAXSEQ, int(nseq[b]), lits.ctypes.data + p0, int(nlit[b]))
        assert r > 0, (case.name, b, r)
        out.append(buf[:r].tobytes())
    return out
