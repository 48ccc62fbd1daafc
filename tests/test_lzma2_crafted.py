"""CPU: conformance of the LZMA2 decoder on hand-built streams (tests/lzma2_craft.py) that choose every feature of the format on
purpose, not only what the encoders happen to write: all 75 (lc, lp, pb) with every literal context and position state, every
chunk kind and the sequences of them no encoder writes (properties changed inside a block, LZMA chunks that go on after a raw one,
state resets), the size limits of a chunk, every packet kind (all four reps, shortrep after each packet kind, matched literals that
mismatch at each bit), overlapping copies, every distance slot up to 51 with every specPos and align value, and the dictionary
bound at its edges; then streams that break one rule each.

The valid corpus is decoded by the oracle (oracle/lzma2_dec_oracle.c), by liblzma -- the check that the writer is independent --
by the reference's Lzma2Decode and its multi-threaded decoder where oracle/_ref is built, and by the kernel sources compiled for
the host (tests/cuemu) with the literal model in shared and in global memory.  The invalid corpus gets the reference's verdict,
which the oracle must share and the emulated kernels must report as corrupt.  The chunk-header walks of the host code
(b200z_lzma2_stream_info and the streaming cut b200z_lzma2_stream_prefix) are checked against what the writer recorded.

Where the reference and liblzma differ: liblzma checks a distance against its own dictionary buffer, which it rounds up, so it is
no arbiter of the dictionary bound; the corpus uses it on valid streams only.
"""
import ctypes
import lzma

import numpy as np
import pytest

import helpers as H
import lzma2_craft as C

CORRUPT = "corrupt"
CONTEXTS = [(lc, lp, pb) for lc in range(9) for lp in range(5) for pb in range(5) if lc + lp <= 4]
TEXT = b"etaoinshrdlucmfwypvbgkjqxz ETAOINSHRDLU.,\n0123456789"


def _text(rng, n):
    return bytes(rng.integers(0, 256, n, dtype=np.uint8).tolist()) if n else b""


def _random_packets(w, rng, n, max_len=40):
    """n valid packets chosen at random in the open chunk: literals (plain and matched), matches of every length class, the four
    reps and shortrep"""
    for _ in range(n):
        room = w.chunk_room()
        if room < 2 or w.pos < 2:
            w.literal(int(rng.integers(256))); continue
        limit = min(w.pos, w.dict_size)
        r = rng.random()
        if r < 0.35:
            w.literal(int(rng.integers(256)) if rng.random() < 0.5 else w.byte_back(w.reps[0] + 1) ^ int(1 << rng.integers(8)))
        elif r < 0.6:
            length = int(rng.choice([2, 3, 4, 5, int(rng.integers(6, 10)), int(rng.integers(10, 18)), int(rng.integers(18, max_len + 18))]))
            w.match(min(length, room, C.MATCH_LEN_MAX), int(rng.integers(1, limit + 1)))
        elif r < 0.9:
            k = int(rng.integers(4))
            if w.reps[k] < w.pos:
                length = int(rng.choice([2, int(rng.integers(3, 10)), int(rng.integers(10, 18)), int(rng.integers(18, max_len + 18))]))
                w.rep(k, min(length, room, C.MATCH_LEN_MAX))
            else:
                w.literal(int(rng.integers(256)))
        else:
            w.shortrep() if w.reps[0] < w.pos else w.literal(65)


def _context_stream(rng, lc, lp, pb):
    """one (lc, lp, pb): every literal context and every position state of isMatch, isRep0Long and the length coders"""
    w = C.Writer(dict_prop=12)
    w.lzma_chunk(0xE0, (lc, lp, pb))
    w.literals(_text(rng, 16 << lp))
    need = ({("lit-ctx", lc, lp, c) for c in range(1 << (lc + lp))} | {("is-match-ps", pb, p) for p in range(1 << pb)} |
            {("rep0-long-ps", pb, p) for p in range(1 << pb)})
    need_len = {(kind, p, cls) for kind in ("match", "rep") for p in range(1 << pb) for cls in range(3)}
    for _ in range(200):
        have_len = {(k[1], k[3], 0 if k[-1] < 10 else (1 if k[-1] < 18 else 2)) for k in w.stats if k[0] == "len"}
        if need <= set(w.stats) and need_len <= have_len:
            break
        _random_packets(w, rng, 40)
        for c in range(1 << (lc + lp)):           # a literal after each top-bits value of the previous byte, at each lp position
            if ("lit-ctx", lc, lp, c) not in w.stats:
                w.literal(int(rng.integers(256)))
    else:
        raise AssertionError((lc, lp, pb))
    w.end_chunk()
    return w


def _overlap_stream():
    """matches of every distance 1..40 with lengths below, equal to and above it, each followed by a matched literal (after an
    overlapping copy its match byte lies inside the copy)"""
    w = C.Writer(dict_prop=16)
    w.lzma_chunk(0xE0, (3, 0, 2))
    w.literals(bytes(range(1, 81)))
    for d in range(1, 41):
        for length in sorted({max(2, d - 1), max(2, d), d + 1, 2 * d + 3, min(273, 7 * d + 5)}):
            w.match(length, d)
            w.literal(w.byte_back(d) ^ 0x10)
    w.end_chunk()
    return w


def _states_stream():
    """a literal from each of the 12 states, shortrep after a literal, a match and a rep, rep1 / rep2 / rep3 each followed by a
    rep0 that shows the rotation, and matched literals whose first mismatch falls at each bit 7..0 (and one with none)"""
    w = C.Writer(dict_prop=16)
    w.lzma_chunk(0xE0, (3, 0, 2))
    w.literals(TEXT * 2)
    w.literal(1)                                                 # state 0
    w.match(3, 7); w.literal(2); w.literal(3); w.literal(4)       # 7, 4, 1
    w.rep(0, 2); w.literal(5); w.literal(6)                      # 8, 5, 2
    w.shortrep(); w.literal(7); w.literal(8)                     # 9, 6, 3
    w.match(4, 9); w.match(5, 31); w.literal(9)                  # 10
    w.match(4, 9); w.rep(1, 3); w.literal(10)                    # 11
    w.literal(11); w.shortrep()                                  # shortrep after a literal
    w.match(6, 17); w.shortrep()                                 # after a match
    w.rep(1, 4); w.shortrep()                                    # after a rep
    w.match(3, 11); w.match(3, 13); w.match(3, 19); w.match(3, 23)
    for k in (1, 2, 3):
        w.rep(k, 2 + k); w.rep(0, 5); w.literal(12 + k)
    w.match(2, 29); w.rep(3, 4); w.rep(3, 3); w.rep(2, 6); w.rep(0, 2)
    for bit in [7, 6, 5, 4, 3, 2, 1, 0, None]:
        w.match(4, 41)
        mb = w.byte_back(w.reps[0] + 1)
        w.literal(mb if bit is None else mb ^ (1 << bit) ^ ((1 << bit) - 1 if bit else 0))
    w.end_chunk()
    return w


def _lengths_stream():
    """lengths 2..5, 9, 10, 17, 18 and 273 for matches and reps at every position state of pb = 2 and pb = 4"""
    out = []
    for pb in (2, 4):
        w = C.Writer(dict_prop=16)
        w.lzma_chunk(0xE0, (0, 0, pb))
        w.literals(TEXT)
        for length in (2, 3, 4, 5, 9, 10, 17, 18, 273):
            for ps in range(1 << pb):
                while w.pos % (1 << pb) != ps:
                    w.literal(0x61)
                w.match(length, 1 + (ps * 7 + length) % 40)
                while w.pos % (1 << pb) != ps:
                    w.literal(0x62)
                w.rep(0, length)
        w.end_chunk()
        out.append((f"lengths-pb{pb}", w))
    return out


def _distance_streams():
    """every specPos value of slots 4..13 and all 16 align values"""
    w = C.Writer(dict_prop=16)
    w.lzma_chunk(0xE0, (0, 0, 0))
    rng = np.random.default_rng(4)
    w.literals(_text(rng, 300))
    for slot in range(4, 14):
        for rem in range(1 << ((slot >> 1) - 1)):
            w.match(2 + rem % 5, C.slot_base(slot) + rem + 1); w.literal(rem & 0xFF)
    w.end_chunk()
    a = C.Writer(dict_prop=18)
    a.lzma_chunk(0xE0, (0, 0, 0))
    a.literals(_text(rng, 5000))
    for rem in range(16):
        for slot in (14, 15, 20, 23):
            a.match(3, C.slot_base(slot) + 16 * (rem * 3 % (1 << ((slot >> 1) - 5))) + rem + 1)
    a.end_chunk()
    return [("spec-pos-slots-4-13", w), ("align-all-16", a)]


def fill_to(w, target, chunk_packets=256):
    """rep0 packets of length 273 at distance 1 up to block position `target`, the last chunk left open: each filler chunk is coded
    afresh until the model has saturated, and from then on repeated"""
    filler = chunk_packets * C.MATCH_LEN_MAX
    while w.pos + filler * 2 + 600 < target:
        w.lzma_chunk(0x80)
        for _ in range(chunk_packets):
            w.rep(0, C.MATCH_LEN_MAX)
        w.end_chunk()
        if w.last_chunk["repeatable"]:
            n = (target - w.pos - 600) // filler - 1
            if n > 0:
                w.repeat_last_chunk(n)
    w.lzma_chunk(0x80)
    while target - w.pos > C.MATCH_LEN_MAX:
        w.rep(0, min(C.MATCH_LEN_MAX, target - w.pos - 2))
    if target - w.pos >= 2:
        w.rep(0, target - w.pos)
    elif target - w.pos == 1:
        w.shortrep()


def far_block(w, rng, slots, head=65536, spread=None):
    """a block that reaches every slot in `slots` with a match back into `head` random literals at its start (the 0xE0 chunk is
    open), and between them the filler of fill_to.  `spread` limits how far above its slot's base a distance lies.  Returns the
    head and [(position, distance, length)] of the far matches; each is followed by a rep1 back to distance 1"""
    assert w.pos == 0
    data = _text(rng, head)
    for i in range(0, head, 1 << 15):                          # random literals pack about 1:1: two chunks
        if i:
            w.lzma_chunk(0x80)
        w.literals(data[i:i + (1 << 15)])
        w.end_chunk()
    far = []
    for slot in slots:
        base = C.slot_base(slot)
        top = C.slot_base(slot + 1) if slot < 63 else 1 << 32
        dist_v = base + int(rng.integers(0, min(top - base, spread or top)))
        lo = max(0, w.pos + 2 - dist_v - 1)                    # the match starts past the current position
        src = int(rng.integers(lo, head - 300))
        target = dist_v + 1 + src
        assert C.dist_slot(dist_v) == slot and target > w.pos
        fill_to(w, target)
        length = int(rng.integers(2, 274))
        w.match(length, dist_v + 1)
        far.append((w.pos - length, dist_v + 1, length))
        w.rep(1, 2 + slot % 7)                                  # back to distance 1
        w.end_chunk()
    return data, far


def valid_corpus():
    """[(name, stream, plaintext, dict_prop, writer)] -- seeded, about 150 streams"""
    rng = np.random.default_rng(20261016)
    V = []

    def add(name, w):
        s, p = w.finish()
        V.append((name, s, p, w.dict_prop, w))

    # ---- every context setting
    for lc, lp, pb in CONTEXTS:
        add(f"ctx-lc{lc}-lp{lp}-pb{pb}", _context_stream(rng, lc, lp, pb))
    # ---- chunk sequences
    w = C.Writer(18); w.lzma_chunk(0xE0, (3, 0, 2)); w.literals(TEXT); _random_packets(w, rng, 200); w.end_chunk()
    for _ in range(2):
        w.lzma_chunk(0x80); _random_packets(w, rng, 200); w.end_chunk()
    add("seq-E0-80-80", w)
    w = C.Writer(18); w.lzma_chunk(0xE0, (1, 1, 1)); w.literals(TEXT); _random_packets(w, rng, 200); w.end_chunk()
    w.lzma_chunk(0xA0); w.rep(0, 5); _random_packets(w, rng, 200); w.end_chunk()   # state reset: rep0 is distance 1
    add("seq-E0-A0-rep0-distance-1", w)
    w = C.Writer(18); w.lzma_chunk(0xE0, (0, 4, 4)); w.literals(TEXT); _random_packets(w, rng, 200); w.end_chunk()
    w.lzma_chunk(0xC0, (4, 0, 0)); _random_packets(w, rng, 200); w.end_chunk()
    w.lzma_chunk(0xC0, (2, 2, 3)); _random_packets(w, rng, 100); w.end_chunk()
    add("seq-E0-C0-C0-new-props", w)
    w = C.Writer(18); w.raw_chunk(TEXT * 3, True); w.lzma_chunk(0xC0, (3, 1, 2)); _random_packets(w, rng, 200); w.end_chunk()
    w.lzma_chunk(0x80); _random_packets(w, rng, 100); w.end_chunk()
    add("seq-1-C0-80", w)
    w = C.Writer(18); w.raw_chunk(TEXT, True); w.raw_chunk(TEXT[::-1], False); w.raw_chunk(b"z", False)
    w.lzma_chunk(0xC0, (0, 2, 1)); _random_packets(w, rng, 200); w.end_chunk()
    add("seq-1-2-2-C0", w)
    for k, (ctl, first) in enumerate([(0x80, "match"), (0x80, "literal"), (0xA0, "literal")]):
        w = C.Writer(18); w.lzma_chunk(0xE0, (3, 0, 2)); w.literals(TEXT); _random_packets(w, rng, 100)
        w.match(7, 20); w.end_chunk()                           # state 7: the next literal is a matched one
        w.raw_chunk(bytes(TEXT[::-1]) * 2, False)
        w.lzma_chunk(ctl)
        w.literal(w.byte_back(w.reps[0] + 1) ^ 0x04)            # match byte inside the raw chunk (rep0 from before it)
        _random_packets(w, rng, 100); w.end_chunk()
        add(f"seq-E0-2-{ctl:02X}-{k}", w)
    w = C.Writer(18); w.lzma_chunk(0xE0, (3, 0, 2)); w.literal(0x42); w.end_chunk()
    add("seq-smallest-lzma-chunk", w)
    w = C.Writer(22); w.lzma_chunk(0xE0, (3, 0, 2)); w.literals(TEXT)
    while w.chunk_room() > 273:
        w.rep(0, 273) if w.chunk_room() % 2 else w.match(273, 1 + w.chunk_room() % 40)
    w.match(w.chunk_room(), 1); w.end_chunk()
    assert w.chunks[-1][2] == C.MAX_UNPACK
    w.raw_chunk(_text(rng, 65536), False)
    add("seq-unpack-2MiB-raw-64KiB-raw-last", w)
    # the largest pack the writer reaches: random literals until one more would overflow 64 KiB
    lits = _text(rng, 70000)
    w = C.Writer(20); w.lzma_chunk(0xE0, (0, 0, 0)); n = 0
    while w.packed_so_far() <= C.MAX_PACK:
        w.literal(lits[n]); n += 1
    w = C.Writer(20); w.lzma_chunk(0xE0, (0, 0, 0)); w.literals(lits[:n - 1]); w.end_chunk()
    assert C.MAX_PACK - 12 < w.chunks[-1][3] - 6 <= C.MAX_PACK
    add("seq-largest-pack", w)
    V.append(("empty", b"\x00", b"", 0, None))
    w = C.Writer(20)
    for b in range(6):
        props = CONTEXTS[int(rng.integers(len(CONTEXTS)))]
        if b % 3 == 2:
            w.raw_chunk(_text(rng, 700), True); w.lzma_chunk(0xC0, props)
        else:
            w.lzma_chunk(0xE0, props)
        w.literals(TEXT); _random_packets(w, rng, 300); w.end_chunk()
    add("blocks-6-own-props", w)
    # rep0 right after a state reset in the middle of a block
    w = C.Writer(18); w.lzma_chunk(0xE0, (3, 0, 2)); w.literals(TEXT); w.match(10, 30); w.end_chunk()
    w.lzma_chunk(0xA0); w.rep(0, 9); w.shortrep(); w.rep(0, 300 - 27); w.end_chunk()
    add("a0-reset-rep0-distance-1", w)
    # ---- packets
    add("states-reps-shortrep-mismatch-bits", _states_stream())
    add("overlap-distances-1-40", _overlap_stream())
    for name, w in _lengths_stream() + _distance_streams():
        add(name, w)
    # ---- the dictionary bound: distance dictSize (rep0 = dictSize - 1) once past it, distance pos before
    for prop in (0, 1, 17):
        ds = C.dict_size(prop)
        for kind in ("match", "rep", "shortrep"):
            w = C.Writer(prop); w.lzma_chunk(0xE0, (3, 0, 2)); w.literals(_text(rng, 40))
            _bound_packet(w, kind, w.pos)
            w.literals(_text(rng, 7))
            _fill_plain(w, rng, ds + 5)
            _bound_packet(w, kind, ds)
            w.end_chunk()
            add(f"dict-bound-prop{prop}-{kind}", w)
    # ---- random mixtures over several chunks and blocks
    for i in range(40):
        w = C.Writer(int(rng.integers(16, 23)))
        for b in range(int(rng.integers(1, 4))):
            props = CONTEXTS[int(rng.integers(len(CONTEXTS)))]
            if rng.random() < 0.3:
                w.raw_chunk(_text(rng, int(rng.integers(1, 3000))), True); w.lzma_chunk(0xC0, props)
            else:
                w.lzma_chunk(0xE0, props)
            for c in range(int(rng.integers(1, 4))):
                if c:
                    r = rng.random()
                    if r < 0.2:
                        w.raw_chunk(_text(rng, int(rng.integers(1, 2000))), False)
                    if r > 0.8:
                        w.lzma_chunk(0xC0, CONTEXTS[int(rng.integers(len(CONTEXTS)))])
                    else:
                        w.lzma_chunk(int(rng.choice([0x80, 0xA0])))
                _random_packets(w, rng, int(rng.integers(1, 500)), max_len=int(rng.choice([20, 273])))
                w.end_chunk()
        add(f"mix-{i}", w)
    return V


def _bound_packet(w, kind, distance):
    """a packet of `kind` at `distance`: a match, a rep1 (after a match that puts the distance in rep1) or a shortrep"""
    if kind == "match":
        w.match(3, distance)
    elif kind == "rep":
        w.match(2, distance); w.match(2, 1); w.rep(1, 4)
    else:
        w.match(2, distance); w.shortrep()


def _fill_plain(w, rng, target):
    """literals and short matches until the block holds `target` bytes"""
    while w.pos < target:
        if target - w.pos > 300 and rng.random() < 0.8:
            w.match(int(rng.integers(100, 274)), int(rng.integers(1, min(w.pos, w.dict_size) + 1)))
        else:
            w.literal(int(rng.integers(256)))


def far_corpus():
    """one block of about 52 MiB whose matches reach every distance slot 0..51 (slot 51 starts at distance 3 * 2^24)"""
    rng = np.random.default_rng(51)
    w = C.Writer(dict_prop=29)
    w.lzma_chunk(0xE0, (0, 0, 0))
    w.literals(_text(rng, 5000))
    for slot in range(0, 24):
        w.match(int(rng.integers(2, 50)), C.slot_base(slot) + 1 + int(rng.integers(0, C.slot_base(slot + 1) - C.slot_base(slot))))
    w.end_chunk()
    # slots 24..51: a second block, each far match reaching back into its random head
    w.lzma_chunk(0xE0, (0, 0, 0))
    far_block(w, rng, range(24, 52), head=65536)
    s, p = w.finish()
    return s, p, w


def invalid_corpus():
    """[(name, stream, dict_prop, verdict)] -- streams that break one rule each"""
    rng = np.random.default_rng(777)
    bad = []

    def start(prop=12, props=(3, 0, 2)):
        w = C.Writer(prop, allow_invalid=True); w.lzma_chunk(0xE0, props); w.literals(TEXT); return w

    def add(name, w, **kw):
        if w.rc is not None:
            w.end_chunk(**kw)
        bad.append((name, w.finish()[0], w.dict_prop, CORRUPT))

    for prop in (0, 1, 17):                                       # one past the dictionary bound, one past the position
        ds = C.dict_size(prop)
        for kind in ("match", "rep", "shortrep"):
            w = start(prop); _fill_plain(w, rng, ds + 5); _bound_packet(w, kind, ds + 1); add(f"dict-bound+1-prop{prop}-{kind}", w)
            w = start(prop); _bound_packet(w, kind, w.pos + 1); add(f"pos-bound+1-prop{prop}-{kind}", w)
    w = C.Writer(12, allow_invalid=True); w.lzma_chunk(0xE0, (3, 0, 2)); w.rep(0, 3); add("rep-at-block-position-0", w, unpack=3)
    w = C.Writer(12, allow_invalid=True); w.lzma_chunk(0xE0, (3, 0, 2)); w.shortrep(); add("shortrep-at-block-position-0", w, unpack=1)
    w = start(); w.end_chunk(); w.lzma_chunk(0xE0); w.rep(2, 4); add("rep-at-block-position-0-of-the-second-block", w, unpack=4)
    w = start(); w.match(10, 20); add("match-one-byte-past-chunk-end", w, unpack=len(TEXT) + 9)
    w = start(); w.match(10, 20); w.rep(0, 6); add("rep-one-byte-past-chunk-end", w, unpack=len(TEXT) + 15)
    w = start(); w.end_marker(); w.literals(b"more"); add("end-marker-mid-chunk", w, unpack=len(TEXT) + 4)
    w = start(); w.end_marker(); add("end-marker-at-chunk-end", w)
    w = start(); add("first-range-byte-not-0", w, first_byte=1)
    w = start(); _random_packets(w, rng, 50); w.end_chunk(pack=w.packed_so_far() + 1); w.stream += b"\x00"   # one byte more, claimed
    add("pack-one-too-large", w)
    w = start(); _random_packets(w, rng, 50); pk = w.packed_so_far(); add("pack-one-too-small", w, pack=pk - 1)
    for x in (1, 0x80):
        w = start(); _random_packets(w, rng, 50); add(f"last-byte-xor-{x:#x}", w, last_byte_xor=x)
    w = start(); _random_packets(w, rng, 50); add("unpack-larger-than-packets", w, unpack=w.total + 1)
    for p in (4, 1):
        w = start(); add(f"pack-{p}", w, pack=p)
    for ctl in (0x80, 0xA0):
        w = C.Writer(12, allow_invalid=True); w.raw_chunk(TEXT, True)
        w.props = (3, 0, 2); w.lzma_chunk(ctl); w.literal(1); add(f"{ctl:02X}-after-ctl1", w)
    # a valid stream decoded with a dictionary one step too small (its largest distance is the dictionary size of its property)
    w = C.Writer(17); w.lzma_chunk(0xE0, (3, 0, 2)); w.literals(TEXT); _fill_plain(w, rng, C.dict_size(17) + 9)
    w.match(5, C.dict_size(17)); w.end_chunk()
    bad.append(("dict-prop-one-step-too-small", w.finish()[0], 16, CORRUPT))
    w = C.Writer(12, allow_invalid=True); w.raw_chunk(TEXT, False); add("raw-ctl2-first", w)
    return bad


# ---------------------------------------------------------------------------------------------------- decoders
@pytest.fixture(scope="module")
def corpus():
    return valid_corpus()


@pytest.fixture(scope="module")
def emu():
    E = H.cuemu_library()
    E.emu_lzma2_decode.restype = ctypes.c_int64
    E.emu_lzma2_decode.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_int]
    return E


def emu_decode(E, comp, prop, cap, glit):
    src = np.frombuffer(comp + bytes(64), dtype=np.uint8); dst = np.zeros(cap + 64, dtype=np.uint8)
    r = E.emu_lzma2_decode(src.ctypes.data, len(comp), prop, dst.ctypes.data, cap, glit)
    return r, dst[:max(r, 0)].tobytes()


def liblzma_decode(comp, prop):
    return lzma.decompress(comp, format=lzma.FORMAT_RAW, filters=[{"id": lzma.FILTER_LZMA2, "dict_size": max(4096, C.dict_size(min(prop, 39)))}])


def oracle_verdict(comp, cap, prop):
    try:
        return H.oracle_lzma2_decompress(comp, cap, prop)
    except ValueError:
        return CORRUPT


def ref_verdict(comp, cap, prop):
    try:
        return H.ref_lzma2_decompress(comp, cap, prop)[0]
    except ValueError:
        return CORRUPT


def test_corpus_covers_the_format(corpus):
    """the coverage is counted from what the writers coded, not assumed"""
    names = [n for n, *_ in corpus]
    assert len(names) == len(set(names)) and len(corpus) >= 140
    st = sum((w.stats for *_, w in corpus if w is not None), C.collections.Counter())
    _, _, fw = far_corpus_cached()
    st = st + fw.stats
    assert {k[1] for k in st if k[0] == "props"} == set(CONTEXTS) and len(CONTEXTS) == 75
    assert {k[1] for k in st if k[0] == "lit-state"} == set(range(12))
    assert {k[1] for k in st if k[0] == "rep"} == {0, 1, 2, 3}
    assert {k[1] for k in st if k[0] == "ctl"} == {0, 1, 2, 0x80, 0xA0, 0xC0, 0xE0}
    assert {k[1] for k in st if k[0] == "slot"} == set(range(52))
    assert {k[1] for k in st if k[0] == "align"} == set(range(16))
    for slot in range(4, 14):
        assert {k[2] for k in st if k[0] == "spec-pos" and k[1] == slot} == set(range(1 << ((slot >> 1) - 1))), slot
    assert {k[1] for k in st if k[0] == "matched-literal-mismatch"} == {None, *range(8)}
    assert {k[1] for k in st if k[0] == "shortrep-after"} >= {"literal", "match", "rep"}
    assert st["unpack", C.MAX_UNPACK] and st["unpack", 1] and any(k[0] == "pack" and k[1] > C.MAX_PACK - 12 for k in st)
    for lc, lp, pb in CONTEXTS:
        w = dict((n, w) for n, *_, w in corpus)[f"ctx-lc{lc}-lp{lp}-pb{pb}"]
        assert {k[3] for k in w.stats if k[0] == "lit-ctx"} == set(range(1 << (lc + lp)))
        assert {k[2] for k in w.stats if k[0] == "is-match-ps"} == set(range(1 << pb))
        assert {k[2] for k in w.stats if k[0] == "rep0-long-ps"} == set(range(1 << pb))
        assert {(k[1], k[3]) for k in w.stats if k[0] == "len"} == {(kind, p) for kind in ("match", "rep") for p in range(1 << pb)}
    for pb in (2, 4):
        w = dict((n, w) for n, *_, w in corpus)[f"lengths-pb{pb}"]
        for length in (2, 9, 10, 17, 18, 273):
            assert {k[3] for k in w.stats if k[0] == "len" and k[-1] == length} == set(range(1 << pb))


def test_writer_is_pinned_by_liblzma_the_oracle_and_the_reference(corpus):
    for name, comp, plain, prop, _ in corpus:
        assert liblzma_decode(comp, prop) == plain, name
        assert H.oracle_lzma2_decompress(comp, len(plain), prop) == (plain, len(comp)), name
        if H.ref_lzma_available():
            assert H.ref_lzma2_decompress(comp, len(plain), prop) == (plain, len(comp)), name
            assert H.ref_lzma2_decompress_mt(comp, len(plain), prop, 4)[0] == plain, name


@pytest.mark.parametrize("glit", [0, 1])
def test_emulated_kernels_decode_the_corpus(corpus, emu, glit):
    for name, comp, plain, prop, _ in corpus:
        assert emu_decode(emu, comp, prop, len(plain), glit) == (len(plain), plain), (name, glit)


_FAR = []


def far_corpus_cached():
    if not _FAR:
        _FAR.append(far_corpus())
    return _FAR[0]


def test_far_distances_to_slot_51():
    comp, plain, w = far_corpus_cached()
    assert len(plain) > 3 << 24 and len(comp) < 4 << 20
    assert liblzma_decode(comp, w.dict_prop) == plain
    assert H.oracle_lzma2_decompress(comp, len(plain), w.dict_prop) == (plain, len(comp))
    if H.ref_lzma_available():
        assert H.ref_lzma2_decompress(comp, len(plain), w.dict_prop)[0] == plain


@pytest.mark.parametrize("glit", [0, 1])
def test_emulated_kernels_far_distances(emu, glit):
    comp, plain, w = far_corpus_cached()
    assert emu_decode(emu, comp, w.dict_prop, len(plain), glit) == (len(plain), plain)


def test_invalid_streams_get_the_reference_verdict(emu):
    """the reference's verdict where it is built, the oracle's pinned one elsewhere; the emulated kernels report corrupt (status 1)
    and so never return bytes"""
    names = [n for n, *_ in invalid_corpus()]
    assert len(names) == len(set(names)) and len(names) >= 35
    for name, comp, prop, verdict in invalid_corpus():
        cap = 1 << 22
        if H.ref_lzma_available():
            assert ref_verdict(comp, cap, prop) == verdict, name
        assert oracle_verdict(comp, cap, prop) == verdict, name
        for glit in (0, 1):
            r, out = emu_decode(emu, comp, prop, cap, glit)
            assert r == -1, (name, glit, r)


# ---------------------------------------------------------------------------------------------------- host walks
def _lib(pkg):
    L = pkg.load_library()
    sz = ctypes.c_size_t
    L.b200z_lzma2_stream_prefix.argtypes = [ctypes.c_void_p, sz, ctypes.c_uint64, ctypes.POINTER(sz), ctypes.POINTER(ctypes.c_uint64),
                                            ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_int)]
    return L


def stream_info(L, comp):
    src = H._np(comp); cs, nb, used = ctypes.c_uint64(), ctypes.c_uint32(), ctypes.c_size_t()
    rc = L.b200z_lzma2_stream_info(src.ctypes.data, len(comp), ctypes.byref(cs), ctypes.byref(nb), ctypes.byref(used))
    return rc, cs.value, nb.value, used.value


def stream_prefix(L, comp, max_content=1 << 62):
    src = H._np(comp); used, cs, nb, ended = ctypes.c_size_t(), ctypes.c_uint64(), ctypes.c_uint32(), ctypes.c_int()
    rc = L.b200z_lzma2_stream_prefix(src.ctypes.data, len(comp), max_content, ctypes.byref(used), ctypes.byref(cs), ctypes.byref(nb), ctypes.byref(ended))
    return rc, used.value, cs.value, nb.value, ended.value


def test_stream_info_counts_blocks(pkg, corpus):
    L = _lib(pkg)
    for name, comp, plain, _, w in corpus:
        assert stream_info(L, comp) == (0, len(plain), len(w.blocks) if w else 0, len(comp)), name


def _header_len(ctl):
    return 3 if ctl <= 2 else (6 if ctl >= 0xC0 else 5)


def test_stream_prefix_cuts_at_block_boundaries(pkg, corpus):
    """at every chunk header +-1 and at 200 seeded cut points of the multi-block streams: the cut lies on a block boundary -- the
    last dictionary-reset header the buffer holds whole, or past the end marker -- counts the plaintext of the blocks before it,
    and the oracle decodes the prefix (with an end marker appended when the stream had not ended) to that plaintext; maxContent
    stops the walk at the first boundary at or beyond it"""
    L = _lib(pkg)
    rng = np.random.default_rng(5)
    multi = [(n, c, p, prop, w) for n, c, p, prop, w in corpus if w and len(w.blocks) > 1]
    assert len(multi) >= 10
    seeded = 0
    for name, comp, plain, prop, w in multi:
        hdr = {o: _header_len(ctl) for o, ctl, *_ in w.chunks}
        points = {o + e for o in hdr for e in (-1, 0, 1)} | {len(comp) - 1, len(comp)}
        extra = {int(x) for x in rng.integers(0, len(comp) + 1, 200 // len(multi) + 1)}
        seeded += len(extra - points)
        for cut in sorted(p for p in points | extra if 0 <= p <= len(comp)):
            rc, used, cs, nb, ended = stream_prefix(L, comp[:cut])
            assert rc == 0, (name, cut)
            if cut == len(comp):
                assert (used, cs, nb, ended) == (len(comp), len(plain), len(w.blocks), 1), (name, cut)
                continue
            k = max(i for i, (s, _) in enumerate(w.blocks) if s + hdr[s] <= cut) if cut >= hdr[0] else 0
            assert (used, cs, nb, ended) == (*w.blocks[k], k, 0), (name, cut, used, cs)
            if used:
                assert H.oracle_lzma2_decompress(comp[:used] + b"\x00", cs, prop) == (plain[:cs], used + 1), (name, cut)
        ends = w.blocks[1:] + [(len(comp), len(plain))]
        for s, d in w.blocks[1:]:
            for mc in (d - 1, d, d + 1):
                first = min((e for e in ends if e[1] >= mc), key=lambda e: e[1])
                assert stream_prefix(L, comp, mc)[1:3] == first, (name, mc)
    assert seeded >= 200


def header_only_stream():
    """one 0xFF chunk (dictionary reset with props) and 2048 chunks of 0x9F: each claims 2 MiB unpacked and 5 bytes packed, with
    a dummy payload -- more than 2^32 bytes in one block"""
    dummy = bytes(5)
    return bytes([0xFF, 0xFF, 0xFF, 0x00, 0x04, 93]) + dummy + (bytes([0x9F, 0xFF, 0xFF, 0x00, 0x04]) + dummy) * 2048 + b"\x00"


def test_block_of_4gib_is_unsupported(pkg):
    L = _lib(pkg)
    rc, cs, nb, _ = stream_info(L, header_only_stream())
    assert rc == -6 and nb == 1 and cs >= 1 << 32
