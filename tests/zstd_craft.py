"""Test support: a small Zstandard frame writer that follows RFC 8878 feature by feature, in plain Python.

It shares no code with any encoder.  Compression ratio does not matter: every choice a frame can make (header field sizes, block
types, literal and sequence modes, table accuracy, normalized counts with "less than 1" entries and zero runs, Huffman weights
stored directly or FSE-compressed, repcodes) is the caller's, so that the decoder's conformance can be tested on frames no encoder
writes.  `Frame.finish()` returns the frame bytes together with the plaintext they encode.

Bitstreams are assembled as lists of (value, nbBits) fields in the order a decoder reads them; `backward_stream` writes them so
that a backward reader (RFC 8878 section 4.1) meets them in that order.
"""
import struct

import numpy as np

# ---------------------------------------------------------------- format tables (RFC 8878 sections 3.1.1.3.2.1.1 and 3.1.1.3.2.2)
LL_BASE = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40, 48, 64,
           0x80, 0x100, 0x200, 0x400, 0x800, 0x1000, 0x2000, 0x4000, 0x8000, 0x10000]
LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
ML_BASE = list(range(3, 35)) + [35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 0x83, 0x103, 0x203, 0x403, 0x803, 0x1003, 0x2003,
                                0x4003, 0x8003, 0x10003]
ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
LL_DEFAULT = [4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1]
ML_DEFAULT = [1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
              1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1]
OF_DEFAULT = [1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1]
DEFAULT = {"ll": (LL_DEFAULT, 6), "of": (OF_DEFAULT, 5), "ml": (ML_DEFAULT, 6)}
MAX_SYM = {"ll": 35, "of": 31, "ml": 52}
MAX_LOG = {"ll": 9, "of": 8, "ml": 9}
MODE = {"pre": 0, "rle": 1, "fse": 2, "rep": 3}
MAGIC = 0xFD2FB528
SKIP_MAGIC = 0x184D2A50
BLOCK_MAX = 131072


def ll_code(v):
    return v if v < 16 else max(c for c in range(36) if LL_BASE[c] <= v)


def ml_code(v):
    return v - 3 if v < 35 else max(c for c in range(53) if ML_BASE[c] <= v)


def of_code(off_base):
    return off_base.bit_length() - 1


def code_of(stream, v):
    """(code, extra value, extra bits) of one sequence field"""
    if stream == "ll":
        c = ll_code(v); return c, v - LL_BASE[c], LL_BITS[c]
    if stream == "ml":
        c = ml_code(v); return c, v - ML_BASE[c], ML_BITS[c]
    c = of_code(v); return c, v - (1 << c), c


def backward_stream(fields):
    """bytes of a backward bitstream whose reader meets `fields` [(value, nbBits), ...] in list order: the fields are written last
    to first from bit 0 up, then the end mark (a 1 bit) and zero padding to the byte"""
    acc, n = 0, 0
    for v, nb in reversed(fields):
        assert 0 <= v < (1 << nb) or (nb == 0 and v == 0), (v, nb)
        acc |= v << n; n += nb
    acc |= 1 << n; n += 1
    return acc.to_bytes((n + 7) // 8, "little")


# ---------------------------------------------------------------- FSE (RFC 8878 section 4.1)
def fse_table(norm, log):
    """decoding table [(symbol, nbBits, baseline)] built the way section 4.1.1 spreads the symbols"""
    size = 1 << log
    assert sum(1 if c == -1 else c for c in norm) == size, (norm, log)
    sym = [None] * size
    high = size - 1
    for s, c in enumerate(norm):
        if c == -1:
            sym[high] = s; high -= 1
    step = (size >> 1) + (size >> 3) + 3
    pos = 0
    for s, c in enumerate(norm):
        for _ in range(max(c, 0)):
            sym[pos] = s
            pos = (pos + step) & (size - 1)
            while pos > high:
                pos = (pos + step) & (size - 1)
    assert pos == 0
    nxt = [1 if c == -1 else c for c in norm]
    tab = []
    for u in range(size):
        s = sym[u]; ns = nxt[s]; nxt[s] += 1
        nb = log - (ns.bit_length() - 1)
        tab.append((s, nb, (ns << nb) - size))
    return tab


class FseCoder:
    """one FSE-coded symbol chain: states are chosen last to first so that each state's successor lies in its range"""

    def __init__(self, norm, log, rle_symbol=None):
        if rle_symbol is not None:
            self.tab, self.log = [(rle_symbol, 0, 0)], 0
        else:
            self.tab, self.log = fse_table(norm, log), log
        self.norm = norm
        self.cover = {}
        for u, (s, nb, base) in enumerate(self.tab):
            c = self.cover.setdefault(s, {})
            for x in range(base, base + (1 << nb)):
                c[x] = u

    def states(self, syms, last_with_bits=False):
        """states for the symbols `syms` (decoder order) and the (value, nbBits) of each transition"""
        cand = [u for u, e in enumerate(self.tab) if e[0] == syms[-1] and (e[1] > 0 or not last_with_bits)]
        assert cand, syms[-1]
        st = [cand[0]]
        for s in reversed(syms[:-1]):
            st.append(self.cover[s][st[-1]])
        st.reverse()
        moves = [(st[k + 1] - self.tab[st[k]][2], self.tab[st[k]][1]) for k in range(len(st) - 1)]
        return st, moves


def write_ncount(norm, log, check=True):
    """FSE table description (section 4.1.1): accuracy log, then the counts with their variable-size fields and zero-run flags.
    check=False writes counts that do not add up to 2^log (a corrupt description)"""
    acc, n = log - 5, 4
    remaining = 1 << log
    s = 0
    while remaining > 0 and s < len(norm):
        v = norm[s] + 1
        nb = (remaining + 1).bit_length()
        T = 1 << (nb - 1); mx = 2 * T - 1 - (remaining + 1)
        if v < mx:
            acc |= v << n; n += nb - 1
        else:
            acc |= (v if v < T else v + mx) << n; n += nb
        remaining -= 1 if norm[s] == -1 else norm[s]
        s += 1
        if v == 1:                                    # a zero count: then 2-bit repeat flags for the zeros after it
            z = 0
            while s + z < len(norm) and norm[s + z] == 0:
                z += 1
            s += z
            while True:
                r = min(z, 3); acc |= r << n; n += 2; z -= r
                if r < 3:
                    break
    assert not check or (remaining == 0 and s == len(norm)), (remaining, s, len(norm))
    return acc.to_bytes((n + 7) // 8, "little")


def make_norm(counts, log, rng=None, less_than_one=0, extra_lt1=0, max_sym=None):
    """normalized counts summing to 2^log over the symbols with counts[s] > 0 (each kept > 0 or -1).  less_than_one: how many of the
    used symbols get the "less than 1" probability (-1); extra_lt1: unused symbols given -1 as well (legal, never coded)"""
    used = [s for s, c in enumerate(counts) if c > 0]
    size = 1 << log
    lt1 = set()
    if rng is not None and less_than_one:
        lt1 = set(rng.choice(used, size=min(less_than_one, len(used) - 1), replace=False).tolist())
    extra = set()
    if rng is not None and extra_lt1 and max_sym is not None:
        free = [s for s in range(max_sym + 1) if s not in used]
        if free:
            extra = set(rng.choice(free, size=min(extra_lt1, len(free)), replace=False).tolist())
    pos = [s for s in used if s not in lt1]
    budget = size - len(lt1) - len(extra)
    assert budget >= len(pos) >= 1, (budget, pos)
    tot = sum(counts[s] for s in pos)
    share = {s: 1 + (counts[s] * (budget - len(pos))) // tot for s in pos}
    share[max(pos, key=lambda s: counts[s])] += budget - sum(share.values())
    top = max(used + list(extra))
    norm = [0] * (top + 1)
    for s in lt1 | extra:
        norm[s] = -1
    for s in pos:
        norm[s] = share[s]
    return norm


# ---------------------------------------------------------------- Huffman (RFC 8878 section 4.2)
def huf_lengths(rng, nsym, max_bits):
    """code lengths of a complete prefix code with `nsym` leaves whose longest code is `max_bits` (nsym > max_bits)"""
    assert 2 <= nsym <= (1 << max_bits) and nsym > max_bits
    lens = [1, 1]
    while max(lens) < max_bits:                           # one deep chain first: the longest code is exactly max_bits
        i = lens.index(max(lens)); d = lens.pop(i); lens += [d + 1, d + 1]
    while len(lens) < nsym:
        cand = [i for i, d in enumerate(lens) if d < max_bits]
        i = cand[int(rng.integers(len(cand)))]; d = lens.pop(i); lens += [d + 1, d + 1]
    rng.shuffle(lens)
    return lens


class Huffman:
    """a literal Huffman table from per-symbol code lengths {symbol: length}; the code of each symbol is where the decoder's
    table (section 4.2.1.5: ranks by weight, symbols in order within a rank) puts it"""

    def __init__(self, lengths):
        self.max_bits = max(lengths.values())
        self.last = max(lengths)
        self.weights = [0] * (self.last + 1)
        for s, ln in lengths.items():
            self.weights[s] = self.max_bits + 1 - ln
        start, pos = {}, 0
        for r in range(1, self.max_bits + 1):
            start[r] = pos
            pos += sum(1 for w in self.weights if w == r) << (r - 1)
        assert pos == 1 << self.max_bits
        self.code = {}
        for s, w in enumerate(self.weights):
            if w:
                nb = self.max_bits + 1 - w
                self.code[s] = (start[w] >> (self.max_bits - nb), nb)
                start[w] += 1 << (w - 1)

    def description(self, direct, fse_log=6):
        """Huffman tree description: the weights of all symbols but the last, as 4-bit values (header byte >= 128) or
        FSE-compressed with two interleaved states (header byte = size)"""
        w = self.weights[:-1]
        if direct:
            assert 1 <= len(w) <= 128
            body = bytes(((w[i] << 4) | (w[i + 1] if i + 1 < len(w) else 0)) for i in range(0, len(w), 2))
            return bytes([127 + len(w)]) + body
        assert len(w) >= 2 and len(set(w)) >= 2, "FSE-compressed weights need two distinct values"
        counts = [0] * 13
        for x in w:
            counts[x] += 1
        norm = make_norm(counts, fse_log)
        fse = FseCoder(norm, fse_log)
        even, odd = w[0::2], w[1::2]
        n = len(w)
        # the state of w[n-2] must read bits when it is updated: that read finds the stream exhausted and ends the weights
        sa, ma = fse.states(even, last_with_bits=(n - 2) % 2 == 0)
        sb, mb = fse.states(odd, last_with_bits=(n - 2) % 2 == 1)
        fields = [(sa[0], fse_log), (sb[0], fse_log)]
        for j in range(n - 2):                            # the update after w[j] moves its state to w[j+2]
            fields.append(ma[j // 2] if j % 2 == 0 else mb[j // 2])
        body = write_ncount(norm, fse_log) + backward_stream(fields)
        assert len(body) < 128, "weights description too long for the FSE form"
        return bytes([len(body)]) + body

    def stream(self, data):
        return backward_stream([self.code[b] for b in data])


# ---------------------------------------------------------------- repcodes and execution (RFC 8878 section 3.1.1.5)
def resolve_offset(reps, off_base, ll):
    """(offset, new repcode history); offset 0 means the "rep0 - 1" repcode gave 0 (corrupt)"""
    if off_base > 3:
        off = off_base - 3
        return off, [off, reps[0], reps[1]]
    idx = off_base - 1 + (ll == 0)
    if idx == 0:
        return reps[0], list(reps)
    off = reps[0] - 1 if idx == 3 else reps[idx]
    if idx == 1:
        return off, [off, reps[0], reps[2]]
    return off, [off, reps[0], reps[1]]


# ---------------------------------------------------------------- frames
def lit_header(ltype, regen, csize=None, sf=None, streams=1):
    """literals section header (section 3.1.1.3.1.1) in the given size format (smallest that fits when sf is None)"""
    if ltype <= 1:
        if sf is None:
            sf = 0 if regen < 32 else (1 if regen < 4096 else 3)
        if sf in (0, 2):
            assert regen < 32; return bytes([ltype | (regen << 3)])
        if sf == 1:
            assert regen < 4096; return struct.pack("<H", ltype | (1 << 2) | (regen << 4))
        assert regen < (1 << 20); v = ltype | (3 << 2) | (regen << 4); return v.to_bytes(3, "little")
    if sf is None:
        big = max(regen, csize)
        sf = (0 if streams == 1 else 1) if big < 1024 else (2 if big < 16384 else 3)
    assert (sf == 0) == (streams == 1)
    if sf <= 1:
        assert regen < 1024 and csize < 1024; return (ltype | (sf << 2) | (regen << 4) | (csize << 14)).to_bytes(3, "little")
    if sf == 2:
        assert regen < 16384 and csize < 16384; return (ltype | (2 << 2) | (regen << 4) | (csize << 18)).to_bytes(4, "little")
    assert regen < (1 << 18) and csize < (1 << 18); return (ltype | (3 << 2) | (regen << 4) | (csize << 22)).to_bytes(5, "little")


def nbseq_header(n, form=None):
    """Number_of_Sequences in its 1-, 2- or 3-byte form (the smallest that fits when form is None)"""
    if form is None:
        form = 1 if n < 128 else (2 if n < 0x7F00 else 3)
    if form == 1:
        assert n < 128; return bytes([n])
    if form == 2:
        assert n < 0x8000; return bytes([128 + (n >> 8), n & 255])
    assert 0x7F00 <= n < 0x7F00 + 0x10000; return bytes([255]) + struct.pack("<H", n - 0x7F00)


def skippable(payload, k=0):
    return struct.pack("<II", SKIP_MAGIC + k, len(payload)) + payload


def size_hint(frame):
    """the 12-byte skippable frame (magic 0x184D2A50, 4 bytes: the compressed size of the frame after it) some writers put before
    each frame so that a reader can find frames without walking their blocks"""
    return skippable(struct.pack("<I", len(frame)))


class Frame:
    """one frame, block by block.  window_log / window_mantissa: the window descriptor (omitted with single=True, where the content
    size is the window); fcs_bytes: 0 (absent), 1 (single-segment only), 2, 4 or 8; dict_id: a dictionary ID field (value, bytes).
    inherit: a Frame whose last Huffman / FSE tables this one may (wrongly) reuse -- for frames that are corrupt on purpose."""

    def __init__(self, window_log=17, window_mantissa=0, single=False, fcs_bytes=None, checksum=False, dict_id=None, inherit=None,
                 fhd_extra=0):
        self.window_log, self.window_mantissa, self.single = window_log, window_mantissa, single
        self.fcs_bytes = (1 if single else 0) if fcs_bytes is None else fcs_bytes
        assert not single or self.fcs_bytes
        self.checksum, self.dict_id, self.fhd_extra = checksum, dict_id, fhd_extra
        self.window = (1 << window_log) + ((1 << window_log) >> 3) * window_mantissa
        self.blocks = []
        self.out = bytearray()
        self.plain_seqs = []                      # (literal length, offset, match length) over the whole plaintext, raw / RLE bytes as literals
        self._pending = 0
        self.reps = [1, 4, 8]
        self.huf = inherit.huf if inherit else None
        self.tables = dict(inherit.tables) if inherit else {}

    # ---- blocks
    def _block(self, btype, size, body, last=False):
        self.blocks.append([btype, size, body, last])

    def raw(self, data, size=None):
        self._block(0, len(data) if size is None else size, bytes(data)); self.out += data; self._pending += len(data)

    def rle(self, byte, n):
        self._block(1, n, bytes([byte])); self.out += bytes([byte]) * n; self._pending += n

    def compressed(self, lits, seqs=(), lit_mode="raw", lit_sf=None, streams=1, huf=None, huf_direct=False, huf_fse_log=6,
                   modes=("fse", "fse", "fse"), logs=(6, 5, 6), rng=None, lt1=(0, 0, 0), extra_lt1=(0, 0, 0), rle_codes=None,
                   nbseq_form=None, check=True, modes_extra=0, lit_regen=None, jump=None, ncount=None, full=(False, False, False)):
        """a compressed block: literal bytes `lits` (raw / rle / huf / treeless) and explicit sequences (ll, offBase, ml).
        modes: LL, OF, ML each 'pre', 'rle', 'fse' or 'rep'; logs: the accuracy logs of the 'fse' ones; lt1 / extra_lt1: "less than 1"
        counts among the used / unused codes.  check=False writes what it is told even where a decoder must refuse it; with it,
        jump replaces the 4-stream jump table and ncount ({'ll' | 'of' | 'ml': bytes}) a table description."""
        lits = bytes(lits)
        seqs = list(seqs)
        if check and seqs:
            for t, k in enumerate(("ll", "of", "ml")):
                if modes[t] == "rep" and (k not in self.tables or any(code_of(k, s[t])[0] not in self.tables[k].cover for s in seqs)):
                    raise ValueError(f"the {k} table to repeat lacks a code")
        # ---- literals section
        regen = len(lits) if lit_regen is None else lit_regen
        if lit_mode == "raw":
            sec = lit_header(0, regen, sf=lit_sf) + lits
        elif lit_mode == "rle":
            assert len(set(lits)) <= 1
            sec = lit_header(1, regen, sf=lit_sf) + lits[:1]
        else:
            desc = b""
            if lit_mode == "huf":
                self.huf = huf
                desc = huf.description(huf_direct, huf_fse_log)
            h = self.huf
            assert h is not None or not check
            if streams == 1:
                body = h.stream(lits)
            else:
                seg = (len(lits) + 3) // 4
                parts = [h.stream(lits[k * seg:(k + 1) * seg]) for k in range(3)] + [h.stream(lits[3 * seg:])]
                sizes = [len(p) for p in parts[:3]] if jump is None else jump
                body = struct.pack("<HHH", *sizes) + b"".join(parts)
            csize = len(desc) + len(body)
            sec = lit_header(2 if lit_mode == "huf" else 3, regen, csize, sf=lit_sf, streams=streams) + desc + body
        # ---- sequences section
        sec += nbseq_header(len(seqs), nbseq_form)
        if seqs:
            names = ("ll", "of", "ml")
            codes = {k: [] for k in names}; extra = {k: [] for k in names}
            for ll, ob, ml in seqs:
                for k, v in zip(names, (ll, ob, ml)):
                    c, x, nb = code_of(k, v)
                    codes[k].append(c); extra[k].append((x, nb))
            modes_byte = modes_extra
            coders = {}
            for t, k in enumerate(names):
                m = modes[t]
                modes_byte |= MODE[m] << (6 - 2 * t)
                if m == "pre":
                    coders[k] = FseCoder(*DEFAULT[k])
                elif m == "rle":
                    sym = codes[k][0] if rle_codes is None else rle_codes[t]
                    assert all(c == sym for c in codes[k]) or not check
                    coders[k] = FseCoder(None, 0, rle_symbol=sym)
                elif m == "fse":
                    cnt = [int(full[t])] * (MAX_SYM[k] + 1)        # full: every code gets a state, so that later blocks may repeat the table
                    for c in codes[k]:
                        cnt[c] += 1
                    lg = logs[t]
                    while (1 << lg) < sum(c > 0 for c in cnt) + extra_lt1[t] and lg < MAX_LOG[k]:     # too many codes for the log asked for
                        lg += 1
                    norm = make_norm(cnt, lg, rng, lt1[t], extra_lt1[t], MAX_SYM[k])
                    coders[k] = FseCoder(norm, lg)
                else:
                    coders[k] = self.tables.get(k) or FseCoder(*DEFAULT[k])      # nothing to repeat (check=False): code with the predefined table
                self.tables[k] = coders[k]
            desc = b""
            for t, k in enumerate(names):
                if modes[t] == "rle":
                    desc += bytes([coders[k].tab[0][0]])
                elif modes[t] == "fse":
                    desc += ncount[k] if ncount and k in ncount else write_ncount(coders[k].norm, coders[k].log)
            st, mv = {}, {}
            for k in names:
                st[k], mv[k] = coders[k].states(codes[k])
            fields = [(st["ll"][0], coders["ll"].log), (st["of"][0], coders["of"].log), (st["ml"][0], coders["ml"].log)]
            for i in range(len(seqs)):
                fields += [extra["of"][i], extra["ml"][i], extra["ll"][i]]
                if i + 1 < len(seqs):
                    fields += [mv["ll"][i], mv["ml"][i], mv["of"][i]]
            sec += bytes([modes_byte]) + desc + backward_stream(fields)
            self.seq_fields = fields                      # (value, nbBits) in reading order: tests may need the bit positions
        # ---- what it decodes to
        lp = 0
        for ll, ob, ml in seqs:
            off, reps = resolve_offset(self.reps, ob, ll)
            self.out += lits[lp:lp + ll]; lp += ll
            if check:
                assert lp <= len(lits) and 0 < off <= min(len(self.out), self.window), (off, len(self.out))
            self.reps = reps
            self.plain_seqs.append((self._pending + ll, off, ml)); self._pending = 0
            if 0 < off <= len(self.out):
                for _ in range(ml):
                    self.out.append(self.out[-off])
        self.out += lits[lp:]; self._pending += len(lits) - lp
        if check:
            assert len(sec) <= BLOCK_MAX
        self._block(2, len(sec), sec)
        return len(sec)

    # ---- the frame
    def header(self):
        fcs_flag = {0: 0, 1: 0, 2: 1, 4: 2, 8: 3}[self.fcs_bytes]
        did_bytes = 0 if self.dict_id is None else self.dict_id[1]
        fhd = (fcs_flag << 6) | (int(self.single) << 5) | (int(self.checksum) << 2) | {0: 0, 1: 1, 2: 2, 4: 3}[did_bytes] | self.fhd_extra
        h = struct.pack("<IB", MAGIC, fhd)
        if not self.single:
            h += bytes([((self.window_log - 10) << 3) | self.window_mantissa])
        if did_bytes:
            h += self.dict_id[0].to_bytes(did_bytes, "little")
        n = len(self.out)
        if self.fcs_bytes == 2:
            assert 256 <= n < 65536 + 256; h += struct.pack("<H", n - 256)
        elif self.fcs_bytes:
            h += n.to_bytes(self.fcs_bytes, "little")
        return h

    def finish(self, last=True, checksum_value=None):
        """(frame bytes, plaintext).  last=False leaves the last block's Last_Block flag clear (a truncated frame)"""
        if not self.blocks:
            self.raw(b"")
        self.blocks[-1][3] = last
        b = bytearray(self.header())
        for btype, size, body, lst in self.blocks:
            b += (int(lst) | (btype << 1) | (size << 3)).to_bytes(3, "little") + body
        if self.checksum:
            if checksum_value is None:
                import helpers
                o = np.frombuffer(bytes(self.out) or b"\0", dtype=np.uint8)
                checksum_value = helpers.oracle().b2zo_xxh64(o.ctypes.data, len(self.out), 0) & 0xFFFFFFFF
            b += struct.pack("<I", checksum_value)
        return bytes(b), bytes(self.out)
