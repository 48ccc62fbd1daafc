"""Test support: a small LZMA2 stream writer in plain Python, written from the LZMA specification.

It shares no code with any encoder.  Compression ratio does not matter: the caller chooses every packet (literal, match, the four
rep kinds, shortrep, end marker) and every chunk (control byte, properties, raw or LZMA, what its header claims), so that the
decoder's conformance can be tested on streams no encoder writes.  `Writer.finish()` returns the stream bytes together with the
plaintext they encode.

A writer made with `keep_plain=False` keeps only the position and the last byte, for streams too large to hold in memory; it then
refuses packets that need the history (matched literals, shortrep).
"""
import collections

PROB_INIT = 1024
TOP = 1 << 24
MAX_UNPACK = 1 << 21
MAX_PACK = 1 << 16
MATCH_LEN_MAX = 273
END_DIST = 0xFFFFFFFF


def dict_size(prop):
    """the dictionary size of the 1-byte LZMA2 coder property (40: 4 GiB - 1)"""
    assert 0 <= prop <= 40
    return 0xFFFFFFFF if prop == 40 else (2 | (prop & 1)) << (prop // 2 + 11)


def dist_slot(dist):
    """distance slot of a distance value (the distance minus one)"""
    if dist < 4:
        return dist
    n = dist.bit_length() - 1
    return (n << 1) | ((dist >> (n - 1)) & 1)


def slot_base(slot):
    """smallest distance value of a slot"""
    return slot if slot < 4 else (2 | (slot & 1)) << ((slot >> 1) - 1)


class RangeEncoder:
    """the LZMA range encoder: 64-bit low, 32-bit range, a pending byte plus a run of 0xFF bytes that a carry may still change"""

    def __init__(self):
        self.low, self.range, self.cache, self.cache_size = 0, 0xFFFFFFFF, 0, 1
        self.out = bytearray()

    def _shift_low(self):
        if self.low < 0xFF000000 or self.low >= 1 << 32:
            carry = self.low >> 32
            temp = self.cache
            while True:
                self.out.append((temp + carry) & 0xFF)
                temp = 0xFF
                self.cache_size -= 1
                if not self.cache_size:
                    break
            self.cache = (self.low >> 24) & 0xFF
        self.cache_size += 1
        self.low = (self.low & 0x00FFFFFF) << 8

    def bit(self, probs, i, b):
        p = probs[i]
        bound = (self.range >> 11) * p
        if b:
            self.low += bound; self.range -= bound; probs[i] = p - (p >> 5)
        else:
            self.range = bound; probs[i] = p + ((2048 - p) >> 5)
        while self.range < TOP:
            self.range <<= 8; self._shift_low()

    def direct(self, v, n):
        for i in range(n - 1, -1, -1):
            self.range >>= 1
            if (v >> i) & 1:
                self.low += self.range
            while self.range < TOP:
                self.range <<= 8; self._shift_low()

    def tree(self, probs, base, v, bits):
        m = 1
        for i in range(bits - 1, -1, -1):
            b = (v >> i) & 1
            self.bit(probs, base + m, b); m = (m << 1) | b

    def tree_rev(self, probs, base, v, bits):
        m = 1
        for i in range(bits):
            b = (v >> i) & 1
            self.bit(probs, base + m, b); m = (m << 1) | b

    def flush(self):
        for _ in range(5):
            self._shift_low()
        return bytes(self.out)

    def flushed_size(self):
        """bytes the chunk would pack if it were flushed now"""
        c = RangeEncoder()
        c.low, c.range, c.cache, c.cache_size = self.low, self.range, self.cache, self.cache_size
        return len(self.out) + len(c.flush())


class LenCoder:
    def __init__(self):
        self.choice = [PROB_INIT, PROB_INIT]                 # choice, choice2
        self.low = [[PROB_INIT] * 8 for _ in range(16)]
        self.mid = [[PROB_INIT] * 8 for _ in range(16)]
        self.high = [PROB_INIT] * 256

    def encode(self, rc, length, ps):
        v = length - 2
        if v < 8:
            rc.bit(self.choice, 0, 0); rc.tree(self.low[ps], 0, v, 3)
        elif v < 16:
            rc.bit(self.choice, 0, 1); rc.bit(self.choice, 1, 0); rc.tree(self.mid[ps], 0, v - 8, 3)
        else:
            rc.bit(self.choice, 0, 1); rc.bit(self.choice, 1, 1); rc.tree(self.high, 0, v - 16, 8)

    def lists(self):
        return [self.choice, self.high] + self.low + self.mid


class Model:
    """the adaptive probabilities of one LZMA state, each set its own list"""

    def __init__(self, lc, lp):
        self.is_match = [[PROB_INIT] * 16 for _ in range(12)]
        self.is_rep = [PROB_INIT] * 12
        self.is_rep_g0 = [PROB_INIT] * 12
        self.is_rep_g1 = [PROB_INIT] * 12
        self.is_rep_g2 = [PROB_INIT] * 12
        self.is_rep0_long = [[PROB_INIT] * 16 for _ in range(12)]
        self.pos_slot = [[PROB_INIT] * 64 for _ in range(4)]
        self.spec_pos = [PROB_INIT] * 115
        self.align = [PROB_INIT] * 16
        self.len = LenCoder()
        self.rep_len = LenCoder()
        self.literal = [PROB_INIT] * (0x300 << (lc + lp))

    def snapshot(self):
        lists = (self.is_match + [self.is_rep, self.is_rep_g0, self.is_rep_g1, self.is_rep_g2] + self.is_rep0_long + self.pos_slot +
                 [self.spec_pos, self.align, self.literal] + self.len.lists() + self.rep_len.lists())
        return tuple(tuple(x) for x in lists)


class Writer:
    """One LZMA2 stream.  Positions, the dictionary bound and the literal contexts count from the last dictionary reset (control
    byte 1 or 0xE0 and above), as the format defines them."""

    def __init__(self, dict_prop=24, keep_plain=True, allow_invalid=False):
        self.dict_prop, self.dict_size = dict_prop, dict_size(dict_prop)
        self.keep_plain, self.allow_invalid = keep_plain, allow_invalid
        self.stream = bytearray()
        self.plain = bytearray()
        self.total = 0                                   # bytes decoded so far
        self.pos = 0                                     # since the last dictionary reset
        self.last = 0                                    # the byte before `pos` (0 at a block start)
        self.props = None
        self.model = None
        self.state, self.reps = 0, [0, 0, 0, 0]
        self.need_init = 0xE0                            # lowest LZMA control byte allowed next
        self.rc = None                                   # the open LZMA chunk's range encoder
        self.chunk = None
        self.chunks = []                                 # (stream offset, control byte, unpack, header + payload bytes)
        self.blocks = []                                 # (stream offset, decoded offset) of each dictionary reset
        self.stats = collections.Counter()
        self.last_kind = None                            # the packet before: "literal", "match", "rep" or "shortrep"

    # ------------------------------------------------------------------------------------------------ helpers
    def _check(self, ok, what):
        if not ok and not self.allow_invalid:
            raise ValueError(what)

    def _emit(self, data):
        if self.keep_plain:
            self.plain += data
        self.total += len(data); self.pos += len(data)
        if data:
            self.last = data[-1]

    def _copy(self, dist, length):
        """append `length` bytes from `dist` back (periodic when they overlap)"""
        if not self.keep_plain:
            self.total += length; self.pos += length; self.last = None
            return
        src = len(self.plain) - dist
        if dist >= length:
            chunk = self.plain[src:src + length]
        else:
            period = self.plain[src:]
            chunk = (period * (length // dist + 1))[:length]
        self._emit(bytes(chunk))

    def byte_back(self, dist):
        """the byte `dist` positions back (1: the last one)"""
        assert self.keep_plain, "this writer keeps no history"
        if dist > len(self.plain):                       # only after an invalid packet (allow_invalid)
            return 0
        return self.plain[len(self.plain) - dist]

    def _ps(self):
        return self.pos & ((1 << self.props[2]) - 1)

    def _open(self):
        assert self.rc is not None, "no LZMA chunk is open"

    def _room(self):
        return MAX_UNPACK - (self.total - self.chunk["start"])

    def _dist_ok(self, rep0, what):
        self._check(rep0 < self.pos, f"{what}: distance {rep0 + 1} beyond the {self.pos} bytes of the block")
        self._check(rep0 < self.dict_size, f"{what}: distance {rep0 + 1} beyond the dictionary ({self.dict_size})")

    # ------------------------------------------------------------------------------------------------ packets
    def literal(self, byte):
        """a literal: matched (against the byte at rep0) after a match, rep or shortrep, plain otherwise"""
        self._open()
        lc, lp, pb = self.props
        ps = self._ps()
        self.stats["lit-state", self.state] += 1
        self.stats["is-match-ps", pb, ps] += 1
        assert self.last is not None or lc == 0, "literal context unknown: this writer keeps no history"
        prev = self.last or 0
        ctx = ((self.pos & ((1 << lp) - 1)) << lc) + (prev >> (8 - lc))
        self.stats["lit-ctx", lc, lp, ctx] += 1
        self.rc.bit(self.model.is_match[self.state], ps, 0)
        probs, base = self.model.literal, 0x300 * ctx
        sym = 1
        if self.state >= 7:
            mb = self.byte_back(self.reps[0] + 1)
            mismatch = None
            for i in range(7, -1, -1):
                b = (byte >> i) & 1
                if mismatch is None:
                    mbit = (mb >> i) & 1
                    self.rc.bit(probs, base + ((1 + mbit) << 8) + sym, b)
                    if mbit != b:
                        mismatch = i
                else:
                    self.rc.bit(probs, base + sym, b)
                sym = (sym << 1) | b
            self.stats["matched-literal-mismatch", mismatch] += 1
        else:
            self.rc.tree(probs, base, byte, 8)
        self.state = 0 if self.state < 4 else (self.state - 3 if self.state < 10 else self.state - 6)
        self.last_kind = "literal"
        self._emit(bytes([byte]))

    def literals(self, data):
        for b in data:
            self.literal(b)

    def _len_ok(self, length, what):
        assert 2 <= length <= MATCH_LEN_MAX, length
        self._check(length <= self._room(), f"{what}: the chunk would decode more than {MAX_UNPACK} bytes")

    def match(self, length, distance):
        """a match of `length` bytes from `distance` back (1 = the last byte); distance END_DIST + 1 is the end marker"""
        self._open()
        dist = distance - 1
        if dist != END_DIST:
            self._dist_ok(dist, "match")
        self._len_ok(length, "match")
        pb = self.props[2]; ps = self._ps()
        self.stats["is-match-ps", pb, ps] += 1
        self.stats["len", "match", pb, ps, min(length - 2, 3), length] += 1
        self.rc.bit(self.model.is_match[self.state], ps, 1)
        self.rc.bit(self.model.is_rep, self.state, 0)
        self.model.len.encode(self.rc, length, ps)
        slot = dist_slot(dist)
        self.stats["slot", slot] += 1
        self.rc.tree(self.model.pos_slot[min(length - 2, 3)], 0, slot, 6)
        if slot >= 4:
            nb = (slot >> 1) - 1
            rem = dist - slot_base(slot)
            if slot < 14:
                self.stats["spec-pos", slot, rem] += 1
                self.rc.tree_rev(self.model.spec_pos, slot_base(slot) - slot - 1, rem, nb)
            else:
                self.stats["align", rem & 15] += 1
                self.rc.direct(rem >> 4, nb - 4)
                self.rc.tree_rev(self.model.align, 0, rem & 15, 4)
        self.state = 7 if self.state < 7 else 10
        self.reps = [dist] + self.reps[:3]
        self.last_kind = "match"
        if dist == END_DIST:
            self.stats["end-marker"] += 1
            return
        self._copy(distance, length)

    def end_marker(self):
        """the LZMA end marker (a match of distance 2^32): LZMA2 chunks have exact sizes and do not allow it"""
        self._check(False, "end marker inside an LZMA2 chunk")
        self.match(2, END_DIST + 1)

    def rep(self, k, length):
        """a match of `length` bytes at the k-th most recent distance (k = 0..3), which becomes rep0"""
        self._open()
        assert 0 <= k <= 3
        self._check(self.pos > 0, "rep at block position 0")
        pb = self.props[2]; ps = self._ps()
        self.stats["is-match-ps", pb, ps] += 1
        self.stats["rep", k] += 1
        self.rc.bit(self.model.is_match[self.state], ps, 1)
        self.rc.bit(self.model.is_rep, self.state, 1)
        if k == 0:
            self.stats["rep0-long-ps", pb, ps] += 1
            self.rc.bit(self.model.is_rep_g0, self.state, 0)
            self.rc.bit(self.model.is_rep0_long[self.state], ps, 1)
        else:
            self.rc.bit(self.model.is_rep_g0, self.state, 1)
            self.rc.bit(self.model.is_rep_g1, self.state, 0 if k == 1 else 1)
            if k > 1:
                self.rc.bit(self.model.is_rep_g2, self.state, 0 if k == 2 else 1)
            self.reps = [self.reps[k]] + self.reps[:k] + self.reps[k + 1:]
        self._dist_ok(self.reps[0], f"rep{k}")
        self._len_ok(length, f"rep{k}")
        self.stats["len", "rep", pb, ps, length] += 1
        self.model.rep_len.encode(self.rc, length, ps)
        self.state = 8 if self.state < 7 else 11
        self.last_kind = "rep"
        self._copy(self.reps[0] + 1, length)

    def shortrep(self):
        """one byte from rep0"""
        self._open()
        self._check(self.pos > 0, "shortrep at block position 0")
        self._dist_ok(self.reps[0], "shortrep")
        self._check(self._room() >= 1, "shortrep beyond the chunk limit")
        pb = self.props[2]; ps = self._ps()
        self.stats["is-match-ps", pb, ps] += 1
        self.stats["rep0-long-ps", pb, ps] += 1
        self.stats["shortrep-after", self.last_kind] += 1
        self.rc.bit(self.model.is_match[self.state], ps, 1)
        self.rc.bit(self.model.is_rep, self.state, 1)
        self.rc.bit(self.model.is_rep_g0, self.state, 0)
        self.rc.bit(self.model.is_rep0_long[self.state], ps, 0)
        self.state = 9 if self.state < 7 else 11
        self.last_kind = "shortrep"
        self._copy(self.reps[0] + 1, 1)

    # ------------------------------------------------------------------------------------------------ chunks
    def _reset_dict(self):
        self.pos, self.last = 0, 0
        self.blocks.append((len(self.stream), self.total))

    def lzma_chunk(self, control, props=None):
        """open an LZMA chunk: 0x80 goes on with the state, 0xA0 resets the state, 0xC0 also sets new properties (lc, lp, pb),
        0xE0 also resets the dictionary"""
        assert self.rc is None, "a chunk is open"
        assert control in (0x80, 0xA0, 0xC0, 0xE0)
        self._check(control >= self.need_init, f"control byte {control:#x} where {self.need_init:#x} or above is required")
        if control >= 0xC0:
            assert props is not None or self.props is not None
            props = tuple(props) if props is not None else self.props
            lc, lp, pb = props
            assert lc + lp <= 4 and pb <= 4 and 0 <= min(props), props
            self.props = props
            self.stats["props", props] += 1
        else:
            assert props is None
        if control == 0xE0:
            self._reset_dict()
        if control >= 0xA0 or self.model is None:
            self.model = Model(*self.props[:2])
            self.state, self.reps = 0, [0, 0, 0, 0]
        self.stats["ctl", control] += 1
        self.need_init = 0
        self.rc = RangeEncoder()
        self.chunk = dict(control=control, start=self.total, pos=self.pos, offset=len(self.stream), snapshot=None)
        if control == 0x80:
            self.chunk["snapshot"] = (self.model.snapshot(), self.state, tuple(self.reps), self.pos)

    def chunk_room(self):
        """bytes the open chunk may still decode"""
        return self._room()

    def packed_so_far(self):
        return self.rc.flushed_size()

    def end_chunk(self, unpack=None, pack=None, first_byte=None, last_byte_xor=0):
        """close the open LZMA chunk and write it with its header.  `unpack` / `pack` replace the sizes the header states,
        `first_byte` the range coder's first byte (always 0), `last_byte_xor` changes the last payload byte"""
        self._open()
        payload = bytearray(self.rc.flush())
        real_unpack = self.total - self.chunk["start"]
        assert (1 if unpack is None else 0) <= real_unpack <= MAX_UNPACK, real_unpack
        assert len(payload) <= MAX_PACK, len(payload)
        if first_byte is not None:
            payload[0] = first_byte
        payload[-1] ^= last_byte_xor
        u = real_unpack if unpack is None else unpack
        p = len(payload) if pack is None else pack
        assert 1 <= u <= MAX_UNPACK and 1 <= p <= MAX_PACK, (u, p)
        ctl = self.chunk["control"]
        hdr = bytes([ctl | ((u - 1) >> 16), ((u - 1) >> 8) & 0xFF, (u - 1) & 0xFF, (p - 1) >> 8, (p - 1) & 0xFF])
        if ctl >= 0xC0:
            lc, lp, pb = self.props
            hdr += bytes([(pb * 5 + lp) * 9 + lc])
        self.chunks.append((len(self.stream), ctl, real_unpack, len(hdr) + len(payload)))
        self.stream += hdr + payload
        self.stats["unpack", real_unpack] += 1
        self.stats["pack", len(payload)] += 1
        snap = self.chunk["snapshot"]
        self.last_chunk = dict(bytes=bytes(hdr + payload), unpack=real_unpack,
                               repeatable=snap is not None and snap[:3] == (self.model.snapshot(), self.state, tuple(self.reps)),
                               plain=bytes(self.plain[len(self.plain) - real_unpack:]) if self.keep_plain else None)
        self.rc = None
        return bytes(hdr + payload)

    def repeat_last_chunk(self, times):
        """write the last LZMA chunk `times` more times.  Valid only for a 0x80 chunk that left the model, the state and the reps as
        it found them (its probabilities have saturated), that reads no literal context and whose size keeps the position classes"""
        c = self.last_chunk
        assert c["repeatable"], "the chunk changed the model: its copies would decode differently"
        assert c["unpack"] % (1 << max(self.props[1], self.props[2])) == 0
        for _ in range(times):
            self.chunks.append((len(self.stream), 0x80, c["unpack"], len(c["bytes"])))
            self.stream += c["bytes"]
            if self.keep_plain:
                self.plain += c["plain"]
            self.total += c["unpack"]; self.pos += c["unpack"]
        self.stats["ctl", 0x80] += times

    def raw_chunk(self, data, reset_dict):
        """an uncompressed chunk (control 1 with a dictionary reset, 2 without)"""
        assert self.rc is None, "a chunk is open"
        assert 1 <= len(data) <= MAX_PACK
        ctl = 1 if reset_dict else 2
        self._check(reset_dict or self.need_init != 0xE0, "raw chunk without a dictionary reset at the start of the stream")
        if reset_dict:
            self._reset_dict()
            self.need_init = 0xC0
        self.stats["ctl", ctl] += 1
        self.chunks.append((len(self.stream), ctl, len(data), 3 + len(data)))
        self.stream += bytes([ctl, (len(data) - 1) >> 8, (len(data) - 1) & 0xFF]) + data
        self._emit(bytes(data))

    def finish(self, end=True):
        """(stream, plaintext); the 0x00 end marker is written unless end=False"""
        assert self.rc is None, "a chunk is open"
        if end:
            self.stats["ctl", 0] += 1
        return bytes(self.stream) + (b"\x00" if end else b""), bytes(self.plain)
