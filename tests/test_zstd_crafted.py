"""CPU: conformance of the Zstandard decoder on hand-built frames (tests/zstd_craft.py) that cover the format feature by feature,
not only what two encoders happen to write: every header field size, raw / RLE / compressed / empty blocks, raw / RLE / Huffman /
treeless literals in 1 and 4 streams and every size format, Huffman weights stored directly and FSE-compressed with codes up to 11
bits, each sequence stream in predefined / RLE / FSE / repeat mode at accuracy logs 5 .. 9/8/9 with "less than 1" counts and zero
runs, explicit repcodes (the rep0 - 1 code included), table reuse across raw / RLE literal blocks and blocks without sequences,
and frames of several 4-block execution units.

The corpus is pinned by the oracle decoder (oracle/zstd_dec_oracle.c) and by the reference decoder where oracle/_ref is built, and
decoded by the kernel sources compiled for the host (tests/cuemu) through the execution units and through stage J.

Rules where RFC 8878 and the reference decoder differ (the oracle and the kernels follow the first column):
  * A 4-stream Huffman literals section whose Regenerated_Size splits into valid stream sizes -- 0, 3 or 4 literals, or 6 or more --
    is valid: RFC 8878 3.1.1.3.1.6 gives the first three streams (size + 3) / 4 literals and the last one the rest.  1, 2 and 5
    literals leave the last stream a negative count and are corrupt.  The reference rejects every 4-stream section of fewer than 6
    literals (MIN_LITERALS_FOR_4_STREAMS); no encoder writes one.
  * An offset larger than the window is corrupt even when that many bytes have been decoded: Window_Size (RFC 8878 3.1.1.1.2) is the
    distance a match may reach back, and a decoder that keeps only the window could not follow it.  The reference only asserts this.
  * No block may be larger than Block_Maximum_Size = min(Window_Size, 128 KiB) (RFC 8878 3.1.1.2.4), neither by its Block_Size field
    (raw, RLE and compressed blocks) nor by what a compressed block decodes to.  The declared window counts, not the content size.
    The reference's streaming decoder enforces both; its one-shot decoder only the size of compressed blocks.  (The oracle and the
    kernels used to accept such blocks.)
"""
import ctypes
import struct

import numpy as np
import pytest

import helpers as H
import zstd_craft as C

# decoder verdicts: oracle return codes and emulator statuses (-B2Z_DERR_*)
CORRUPT, UNSUPPORTED, CHECKSUM = "corrupt", "unsupported", "checksum"
ORACLE_RC = {-1: CORRUPT, -3: CHECKSUM, -4: UNSUPPORTED}
EMU_RC = {-1: CORRUPT, -2: UNSUPPORTED, -16: CHECKSUM}


def _lits(rng, n, alphabet):
    """n literal bytes over `alphabet`, skewed so that code lengths differ"""
    a = np.asarray(list(alphabet), dtype=np.uint8)
    p = 1.0 / np.arange(1, len(a) + 1) ** 1.1
    return bytes(rng.choice(a, size=n, p=p / p.sum()).tolist())


def _huf(rng, lits, max_bits, extra=()):
    syms = sorted(set(lits) | set(extra))
    return C.Huffman(dict(zip(syms, C.huf_lengths(rng, len(syms), max_bits))))


def _seqs(rng, fr, nlits, nseq, ml_max=40, rep=0.5, far=None, ll0=0.2):
    """nseq valid sequences for frame `fr` that use at most nlits literals: repcodes (all three, and rep0 - 1 with ll = 0) about
    `rep` of the time, real offsets up to what has been produced and the window (or within `far` of the window when given).  The
    block they make stays within Block_Maximum_Size"""
    out = []
    produced, reps, left = len(fr.out), list(fr.reps), nlits
    room = min(fr.window, C.BLOCK_MAX) - nlits                   # match bytes the block can still take
    for _ in range(nseq):
        ll = 0 if (rng.random() < ll0 or left == 0) else int(rng.integers(1, min(left, 24) + 1))
        if produced + ll == 0:
            ll = min(left, 1)
        if produced + ll == 0:
            break
        avail = min(produced + ll, fr.window)
        ob = int(rng.integers(1, 4)) if rng.random() < rep else 0
        if ob:
            off, nreps = C.resolve_offset(reps, ob, ll)
            if not 0 < off <= avail:
                ob = 0
        if not ob:
            lo = max(1, avail - far) if far else 1
            off = int(rng.integers(lo, avail + 1)); ob = off + 3
            off, nreps = C.resolve_offset(reps, ob, ll)
        ml = min(int(rng.integers(3, ml_max + 1)), room)
        if ml < 3:
            break
        room -= ml
        out.append((ll, ob, ml)); produced += ll + ml; left -= ll; reps = nreps
    return out


TEXT = b"etaoinshrdlucmfwypvbgkjqxz ETAOINSHRDLU.,\n0123456789"


def valid_corpus():
    """[(name, frame, plaintext, reference_accepts)] -- seeded, about 100 frames"""
    rng = np.random.default_rng(20261016)
    V = []

    def add(name, fr, ref_ok=True):
        comp, plain = fr.finish()
        V.append((name, comp, plain, ref_ok))

    # ---- frame headers: content-size field sizes, single segment, window descriptors, checksum
    for fcs, single, wl, wm, ck, n in [(0, False, 10, 0, False, 100), (1, True, 0, 0, False, 200), (2, True, 0, 0, True, 256), (2, False, 17, 3, False, 65791),
                                       (4, True, 0, 0, False, 3000), (4, False, 17, 7, True, 70000), (8, True, 0, 0, True, 5000), (8, False, 20, 1, False, 1),
                                       (0, False, 25, 5, True, 0), (1, True, 0, 0, True, 0), (2, False, 10, 0, False, 300)]:
        fr = C.Frame(window_log=wl or 10, window_mantissa=wm, single=single, fcs_bytes=fcs, checksum=ck)
        data = _lits(rng, n, TEXT)
        if n > 300:
            lits = data[:n // 3]; fr.raw(data[n // 3: n // 2]); rest = n - n // 2
            seqs = _seqs(rng, fr, len(lits), 10, ml_max=max(3, rest // 12))
            fr.compressed(lits, seqs, lit_mode="huf", huf=_huf(rng, lits, 8), streams=4)
            fr.raw(_lits(rng, n - len(fr.out), TEXT))
        elif n:
            fr.raw(data)
        add(f"hdr-fcs{fcs}-single{int(single)}-w{wl}.{wm}-ck{int(ck)}-n{n}", fr)
    # ---- blocks: raw / RLE / compressed up to 128 KiB, empty last block
    fr = C.Frame(window_log=18, fcs_bytes=4); fr.raw(_lits(rng, C.BLOCK_MAX, TEXT)); fr.rle(7, C.BLOCK_MAX); fr.raw(b""); add("blocks-full-raw-rle-empty-last", fr)
    fr = C.Frame(window_log=18, checksum=True); fr.rle(0, 1); fr.raw(b"x")
    lits = _lits(rng, 2000, TEXT); fr.compressed(lits, [(10, 4, 65536), (0, 1, 60000)] + _seqs(rng, fr, 0, 0), lit_mode="raw")
    fr.raw(b""); add("blocks-compressed-128k-regen", fr)
    # ---- literals: every type, stream count and size format
    for ltype, sf, n in [("raw", 0, 31), ("raw", 2, 17), ("raw", 1, 4095), ("raw", 3, 5), ("raw", 3, 100000), ("rle", 0, 9), ("rle", 1, 2000),
                         ("rle", 3, 120000), ("rle", 3, 1)]:
        fr = C.Frame(window_log=17, fcs_bytes=4); fr.raw(b"prefix bytes")
        lits = _lits(rng, n, TEXT) if ltype == "raw" else bytes([0x41]) * n
        fr.compressed(lits, _seqs(rng, fr, n, 5), lit_mode=ltype, lit_sf=sf)
        add(f"lit-{ltype}-sf{sf}-n{n}", fr)
    for streams, sf, n, mb, direct in [(1, 0, 1023, 5, True), (1, 0, 1, 1, True), (4, 1, 1023, 9, False), (4, 2, 1024, 11, True), (4, 2, 12000, 11, False),
                                       (4, 3, 16384, 10, True), (4, 3, 120000, 11, False), (4, 1, 6, 2, True), (4, 1, 7, 3, False), (1, 0, 2, 1, False)]:
        fr = C.Frame(window_log=17, fcs_bytes=8)
        alpha = TEXT if mb > 5 else TEXT[:mb + 2]
        lits = _lits(rng, n, alpha)
        extra = list(range(60, 60 + (13 if mb >= 11 else 0)))
        syms = sorted(set(lits) | set(extra))
        if len(syms) <= mb:
            syms += [s for s in range(1, 128) if s not in syms][:mb + 1 - len(syms)]
        h = C.Huffman(dict(zip(syms, C.huf_lengths(rng, len(syms), mb)))) if len(syms) > 1 else None
        if h is None or (not direct and len(set(h.weights[:-1])) < 2):
            direct = True
        fr.compressed(lits, _seqs(rng, fr, n, 20), lit_mode="huf", huf=h, huf_direct=direct, streams=streams, lit_sf=sf)
        add(f"lit-huf-{streams}s-sf{sf}-n{n}-mb{mb}-{'direct' if direct else 'fse'}", fr)
    # 4 streams with 0, 3 and 4 literals: valid by RFC 8878, refused by the reference (see the module docstring)
    for n in (0, 3, 4):
        fr = C.Frame(window_log=12, fcs_bytes=2); fr.raw(b"z" * 300)
        lits = b"abca"[:n]
        fr.compressed(lits, [(n, 7, 40)], lit_mode="huf", huf=_huf(rng, b"abc", 2), huf_direct=True, streams=4, lit_sf=1)
        add(f"lit-huf-4s-n{n}-rfc", fr, ref_ok=False)
    # offset equal to the window (1 KiB) after 3000 bytes: the largest a match may reach back (invalid twin: offset-beyond-window)
    fr = C.Frame(window_log=10, fcs_bytes=0)
    for k in range(3):
        fr.raw(_lits(rng, 1000, TEXT))
    fr.compressed(b"xyz", [(3, 3 + 1024, 10)])
    add("offset-equals-window", fr)
    # treeless literals after raw and after RLE literal blocks, and across raw / RLE blocks
    fr = C.Frame(window_log=17, fcs_bytes=4, checksum=True)
    lits = _lits(rng, 3000, TEXT); h = _huf(rng, lits, 10)
    fr.compressed(lits, _seqs(rng, fr, 3000, 30), lit_mode="huf", huf=h, streams=4)
    fr.compressed(lits[:500], _seqs(rng, fr, 500, 8), lit_mode="raw")
    fr.compressed(lits[:700], _seqs(rng, fr, 700, 8), lit_mode="treeless", streams=4)
    fr.compressed(b"q" * 90, _seqs(rng, fr, 90, 4), lit_mode="rle")
    fr.raw(b"raw block between"); fr.rle(9, 1000)
    fr.compressed(lits[1000:1400], _seqs(rng, fr, 400, 8), lit_mode="treeless", streams=1)
    fr.compressed(lits[5:2005], [], lit_mode="treeless", streams=4, lit_sf=2)
    add("lit-treeless-after-raw-rle", fr)
    # ---- sequences: modes, accuracy logs, "less than 1" counts, zero runs, Number_of_Sequences forms
    combos = [("pre", "pre", "pre"), ("rle", "rle", "rle"), ("fse", "fse", "fse"), ("fse", "pre", "rle"), ("rle", "fse", "pre"), ("pre", "rle", "fse")]
    logs_list = [(5, 5, 5), (9, 8, 9), (6, 5, 6), (7, 6, 8), (8, 7, 5), (5, 8, 9)]
    for k, modes in enumerate(combos):
        for j, logs in enumerate(logs_list[k % 3::3]):
            fr = C.Frame(window_log=16, fcs_bytes=4, checksum=bool(j))
            fr.raw(_lits(rng, 5000, TEXT))
            lits = _lits(rng, 4000, TEXT)
            if "rle" in modes:
                # one code per RLE stream: ll in one LL code, offsets in one OF code, ml in one ML code
                ll_pick, ml_pick = int(rng.integers(0, 16)), int(rng.integers(3, 35))
                base = 1 << int(rng.integers(4, 12)); seqs = []
                for _ in range(40):
                    ll = ll_pick if modes[0] == "rle" else int(rng.integers(0, 20))
                    ml = ml_pick if modes[2] == "rle" else int(rng.integers(3, 200))
                    ob = (base + int(rng.integers(0, base))) if modes[1] == "rle" else int(rng.integers(4, 4000))
                    seqs.append((ll, ob, ml))
                seqs = [s for s in seqs][:max(1, min(40, 4000 // max(1, ll_pick)))]
            else:
                seqs = _seqs(rng, fr, 4000, 120, ml_max=12 if min(logs) == 5 else 300)     # accuracy log 5: few enough codes for 32 states
            fr.compressed(lits, seqs, modes=modes, logs=logs, rng=rng, lt1=(2, 2, 2), extra_lt1=(3, 2, 4), lit_mode="huf", huf=_huf(rng, lits, 11), streams=4)
            add(f"seq-{'-'.join(modes)}-logs{'.'.join(map(str, logs))}", fr)
    for form, n in [(1, 127), (2, 5), (2, 128), (2, 0x7EFF), (3, 0x7F00), (3, 32767 + 100)]:
        fr = C.Frame(window_log=17, fcs_bytes=4); fr.raw(b"ab")
        seqs = [(1, 4, 3)] + [(0, 1, 3)] * (n - 1) if n > 200 else _seqs(rng, fr, 600, n, ml_max=20)     # offset 1, then repcode 1 (= rep1, ll = 0)
        fr.compressed(_lits(rng, 600, TEXT), seqs, lit_mode="raw", nbseq_form=form, modes=("fse", "fse", "pre") if n > 200 else ("fse",) * 3, logs=(5, 5, 5), rng=rng)
        add(f"seq-count-form{form}-n{n}", fr)
    # zero sequences in every count form, then repeat mode: tables come from the last block that HAD sequences
    fr = C.Frame(window_log=17, fcs_bytes=4)
    lits = _lits(rng, 2000, TEXT)
    fr.compressed(lits, _seqs(rng, fr, 2000, 50), modes=("fse", "fse", "fse"), logs=(7, 6, 7), rng=rng, lt1=(1, 1, 1), full=(True,) * 3)
    fr.compressed(lits[:50], [], lit_mode="raw")
    fr.compressed(lits[:50], [], lit_mode="raw", nbseq_form=2)
    fr.compressed(lits[50:450], _seqs(rng, fr, 400, 30), modes=("rep", "rep", "rep"))
    add("seq-repeat-after-zero-sequences", fr)
    # repeat mode whose source block used RLE (and predefined) mode
    for src_modes in [("rle", "rle", "rle"), ("pre", "rle", "pre"), ("rle", "pre", "fse")]:
        fr = C.Frame(window_log=17, fcs_bytes=4); fr.raw(_lits(rng, 3000, TEXT))
        seqs = [(2, 1000 + 3 if src_modes[1] == "rle" else int(rng.integers(4, 2000)), 5 if src_modes[2] == "rle" else int(rng.integers(3, 50)))
                for _ in range(20)]
        seqs = [((2 if src_modes[0] == "rle" else int(rng.integers(0, 5))), ob, ml) for _, ob, ml in seqs]
        fr.compressed(_lits(rng, 200, TEXT), seqs, modes=src_modes, logs=(6, 5, 6), rng=rng)
        fr.compressed(_lits(rng, 200, TEXT), seqs[:7], modes=("rep", "rep", "rep"))
        fr.compressed(_lits(rng, 100, TEXT), [], lit_mode="raw")
        fr.compressed(_lits(rng, 200, TEXT), seqs[3:9], modes=("rep", "rep", "rep"))
        add(f"seq-repeat-after-{'-'.join(src_modes)}", fr)
    # repcodes chosen explicitly: every repcode with ll = 0 and ll > 0, rep0 - 1, repeated offsets
    fr = C.Frame(window_log=17, fcs_bytes=4, checksum=True); fr.raw(_lits(rng, 200, TEXT))
    seqs = [(3, 13, 4), (2, 23, 5), (1, 53, 6), (0, 1, 4), (0, 2, 4), (0, 3, 4), (0, 3, 4), (4, 1, 3), (5, 2, 3), (6, 3, 3), (0, 3, 9), (0, 1, 3), (1, 1, 3)]
    fr.compressed(_lits(rng, 40, TEXT), seqs, modes=("pre", "pre", "pre"))
    fr.compressed(_lits(rng, 40, TEXT), [(0, 3, 5), (0, 2, 5), (2, 3, 5), (0, 3, 5)], modes=("fse", "fse", "fse"), logs=(5, 5, 5), rng=rng)
    add("seq-repcodes-explicit", fr)
    # ---- frames of several 4-block execution units, matches that reach back across units, mixed block types
    for nb in (3, 4, 5, 8, 9, 13):
        fr = C.Frame(window_log=22, fcs_bytes=4 if nb % 2 else 0, checksum=nb > 8)
        lits_all = _lits(rng, 200000, TEXT); h = _huf(rng, lits_all[:5000], 11)
        for b in range(nb):
            kind = b % 5
            if kind == 3:
                fr.rle(int(rng.integers(256)), int(rng.integers(1, 60000)))
            elif kind == 4:
                fr.raw(lits_all[:int(rng.integers(1, 9000))])
            else:
                lits = lits_all[b * 3000:(b + 1) * 3000]
                seqs = _seqs(rng, fr, len(lits), 200, ml_max=400, far=1 << 20)
                fr.compressed(lits, seqs, lit_mode=("huf", "treeless", "raw")[kind] if b else "huf", huf=h, streams=4,
                              modes=("fse", "fse", "fse") if b == 0 else (("rep", "fse", "rep") if kind == 1 else ("fse", "rep", "pre")), logs=(9, 8, 9), rng=rng,
                              full=(True,) * 3)
        add(f"units-{nb}-blocks", fr)
    # ---- random mixtures
    for i in range(30):
        fr = C.Frame(window_log=int(rng.integers(17, 22)), window_mantissa=int(rng.integers(8)), fcs_bytes=int(rng.choice([0, 4, 8])), checksum=bool(rng.random() < .5))
        have_huf = False; have_tab = False
        for b in range(int(rng.integers(1, 7))):
            r = rng.random()
            if r < .15:
                fr.raw(_lits(rng, int(rng.integers(0, 3000)), TEXT)); continue
            if r < .25:
                fr.rle(int(rng.integers(256)), int(rng.integers(0, 5000))); continue
            n = int(rng.integers(0, 5000)); lits = _lits(rng, n, TEXT if rng.random() < .7 else bytes(range(0, 256, 3)))
            lm = rng.choice(["raw", "rle", "huf", "treeless"]) if n >= 8 else "raw"
            if lm == "rle":
                lits = lits[:1] * n
            if lm == "treeless" and not (have_huf and set(lits) <= set(fr.huf.code)):
                lm = "huf"
            h = None
            if lm == "huf":
                syms = sorted(set(lits))
                if len(syms) < 2:
                    lm = "raw"
                else:
                    mb = int(rng.integers(max(2, len(syms).bit_length()), 12)) if len(syms) < 2048 else 11
                    mb = max(mb, 1)
                    if len(syms) <= mb:
                        syms += [s for s in range(256) if s not in syms][:mb + 1 - len(syms)]
                    h = C.Huffman(dict(zip(syms, C.huf_lengths(rng, len(syms), mb)))); have_huf = True
            streams = 4 if (lm in ("huf", "treeless") and n >= 6 and rng.random() < .6) else 1
            if streams == 1 and lm in ("huf", "treeless") and n >= 1024:
                streams = 4
            seqs = _seqs(rng, fr, n, int(rng.integers(0, 300)), ml_max=int(rng.choice([10, 100, 1000])), far=int(rng.choice([64, 1 << 20])))
            modes = tuple(rng.choice(["pre", "fse", "rep"] if have_tab else ["pre", "fse"]) for _ in range(3))
            direct = bool(rng.random() < .5)
            if h is not None and (h.last > 128 or len(set(h.weights[:-1])) < 2):
                direct = h.last <= 128                  # 4-bit weights cover 128 symbols, the FSE form needs two weight values
                if not direct and len(set(h.weights[:-1])) < 2:
                    lm, h = "raw", None
            kw = dict(lit_mode=str(lm), huf=h, huf_direct=direct, streams=streams if lm in ("huf", "treeless") else 1,
                      logs=(int(rng.integers(5, 10)), int(rng.integers(5, 9)), int(rng.integers(5, 10))), rng=rng,
                      lt1=tuple(int(x) for x in rng.integers(0, 3, 3)), extra_lt1=tuple(int(x) for x in rng.integers(0, 3, 3)))
            try:
                fr.compressed(lits, seqs, modes=modes, **kw)
            except ValueError:                          # a table to repeat that lacks one of the codes: describe it afresh
                fr.compressed(lits, seqs, modes=tuple("fse" if m == "rep" else m for m in modes), **kw)
            have_tab = have_tab or bool(seqs)
        add(f"mix-{i}", fr)
    return V


def invalid_corpus():
    """[(name, stream, verdict)] -- frames the decoders must refuse, and how"""
    rng = np.random.default_rng(777)
    bad = []

    def base():
        fr = C.Frame(window_log=16, fcs_bytes=4); fr.raw(_lits(rng, 3000, TEXT)); return fr

    # offsets: beyond the bytes produced so far, beyond the window (with the bytes there), rep0 - 1 = 0
    fr = C.Frame(window_log=12, fcs_bytes=0); fr.raw(b"a" * 100)
    fr.compressed(b"xyz", [(3, 3 + 104, 10)], check=False); bad.append(("offset-beyond-output", fr.finish()[0], CORRUPT))
    fr = C.Frame(window_log=10, fcs_bytes=0)                    # 3000 bytes in raw blocks that fit the 1 KiB window, then offset 1025
    for k in range(3):
        fr.raw(_lits(rng, 1000, TEXT))
    fr.compressed(b"xyz", [(3, 3 + 1025, 10)], check=False); bad.append(("offset-beyond-window", fr.finish()[0], CORRUPT))
    fr = base(); fr.compressed(b"xyz", [(3, 1 + 3, 10), (0, 1, 5), (0, 3, 4)], check=False); bad.append(("rep0-minus-1-is-zero", fr.finish()[0], CORRUPT))
    # literal lengths beyond the literals section
    fr = base(); fr.compressed(b"abcdef", [(4, 10, 5), (3, 1, 5)], check=False); bad.append(("literal-lengths-beyond-literals", fr.finish()[0], CORRUPT))
    # 4 streams with 1, 2 and 5 literals: a negative last stream
    for n in (1, 2, 5):
        fr = base(); lits = b"abcab"[:n]
        fr.compressed(lits, [], lit_mode="huf", huf=_huf(rng, b"abc", 2), huf_direct=True, streams=4, lit_sf=1, check=False)
        bad.append((f"4-streams-{n}-literals", fr.finish()[0], CORRUPT))
    # jump table sizes that do not match the streams
    fr = base(); lits = _lits(rng, 400, TEXT)
    fr.compressed(lits, [], lit_mode="huf", huf=_huf(rng, lits, 8), streams=4, jump=[1, 1, 1], check=False); bad.append(("jump-table-mismatch", fr.finish()[0], CORRUPT))
    fr = base()
    fr.compressed(lits, [], lit_mode="huf", huf=_huf(rng, lits, 8), streams=4, jump=[60000, 1, 1], check=False); bad.append(("jump-table-beyond", fr.finish()[0], CORRUPT))
    # table reuse with nothing to reuse: the first compressed block of a frame, after a frame that did define tables
    prev = base(); lits = _lits(rng, 400, TEXT)
    prev.compressed(lits, _seqs(rng, prev, 400, 10), lit_mode="huf", huf=_huf(rng, lits, 9), streams=4, logs=(6, 6, 6), rng=rng, full=(True,) * 3)
    good, _ = prev.finish()
    fr = C.Frame(window_log=16, fcs_bytes=4, inherit=prev); fr.raw(lits)
    fr.compressed(lits[:100], [], lit_mode="treeless", streams=1, check=False); bad.append(("treeless-from-previous-frame", good + fr.finish()[0], CORRUPT))
    fr = C.Frame(window_log=16, fcs_bytes=4, inherit=prev); fr.raw(lits)
    fr.compressed(lits[:100], [(1, 1, 4), (2, 1, 3)], modes=("rep", "pre", "pre"), check=False); bad.append(("repeat-from-previous-frame", good + fr.finish()[0], CORRUPT))
    fr = C.Frame(window_log=16, fcs_bytes=4); fr.raw(lits)
    fr.compressed(lits[:100], [(1, 1, 4)], modes=("pre", "pre", "rep"), check=False); bad.append(("repeat-first-block", fr.finish()[0], CORRUPT))
    # repeat mode after blocks without sequences only
    fr = C.Frame(window_log=16, fcs_bytes=4); fr.raw(lits); fr.compressed(lits[:10], [])
    fr.compressed(lits[:100], [(1, 1, 4)], modes=("rep", "rep", "rep"), check=False); bad.append(("repeat-after-zero-sequences-only", fr.finish()[0], CORRUPT))
    # a normalized-count header that does not sum to the table size, Huffman weights that are not a power of two
    fr = base(); seqs = _seqs(rng, fr, 100, 10)
    short = C.write_ncount([1] * 53, 6, check=False)                 # 53 ML codes of count 1 leave 11 of the 64 states unassigned
    fr.compressed(lits[:100], seqs, modes=("pre", "pre", "fse"), logs=(6, 5, 6), rng=rng, ncount={"ml": short}, check=False)
    bad.append(("ncount-bad-sum", fr.finish()[0], CORRUPT))
    fr = base(); h = C.Huffman({97: 1, 98: 2, 99: 3, 100: 3})
    h.weights = [0] * 97 + [3, 3, 1, 1]     # explicit weights 3, 3, 1: 4 + 4 + 1 = 9, and 16 - 9 = 7 is no power of two
    fr.compressed(b"abcd" * 10, [], lit_mode="huf", huf=h, huf_direct=True, streams=1, check=False); bad.append(("huffman-weights-not-power-of-two", fr.finish()[0], CORRUPT))
    # block headers: larger than the limit, reserved type, missing last block; frame header reserved bit; modes reserved bits
    fr = C.Frame(window_log=20, fcs_bytes=0); fr.raw(b"x" * (C.BLOCK_MAX + 1)); bad.append(("raw-block-over-limit", fr.finish()[0], CORRUPT))
    fr = C.Frame(window_log=20, fcs_bytes=0); fr.rle(1, C.BLOCK_MAX + 1); bad.append(("rle-block-over-limit", fr.finish()[0], CORRUPT))
    comp, _ = base().finish(); b = bytearray(comp); b[6 + 4] |= 6; bad.append(("block-type-reserved", bytes(b), CORRUPT))
    # Block_Maximum_Size is min(Window_Size, 128 KiB): raw, RLE and compressed blocks larger than a 1 KiB window
    fr = C.Frame(window_log=10, fcs_bytes=0); fr.raw(b"x" * 1025); bad.append(("raw-block-over-window", fr.finish()[0], CORRUPT))
    fr = C.Frame(window_log=10, fcs_bytes=0); fr.rle(3, 1025); bad.append(("rle-block-over-window", fr.finish()[0], CORRUPT))
    fr = C.Frame(window_log=10, fcs_bytes=0); fr.raw(b"y" * 1000); fr.compressed(b"abc", [(3, 4, 1100)]); bad.append(("compressed-block-decodes-over-window", fr.finish()[0], CORRUPT))
    fr = base(); fr.raw(b"tail"); bad.append(("missing-last-block", fr.finish(last=False)[0], CORRUPT))
    fr = C.Frame(window_log=16, fcs_bytes=4, fhd_extra=8); fr.raw(b"abc"); bad.append(("frame-header-reserved-bit", fr.finish()[0], CORRUPT))
    fr = C.Frame(window_log=32, fcs_bytes=4); fr.raw(b"abc"); bad.append(("window-exponent-over-31", fr.finish()[0], CORRUPT))     # descriptor 0xB0
    fr = base(); fr.compressed(b"abc", [(3, 8, 5)], modes_extra=1, check=False); bad.append(("modes-reserved-bits", fr.finish()[0], CORRUPT))
    # content size and checksum
    fr = C.Frame(window_log=16, fcs_bytes=4); fr.raw(b"abc"); comp, _ = fr.finish(); b = bytearray(comp); b[6] += 1; bad.append(("content-size-mismatch", bytes(b), CORRUPT))
    fr = C.Frame(window_log=16, fcs_bytes=4, checksum=True); fr.raw(b"abcdef"); comp, _ = fr.finish(checksum_value=12345); bad.append(("checksum-mismatch", comp, CHECKSUM))
    # a dictionary ID (1, 2 and 4-byte fields): unsupported
    for nbytes in (1, 2, 4):
        fr = C.Frame(window_log=16, fcs_bytes=4, dict_id=(0x5A, nbytes)); fr.raw(b"abc"); bad.append((f"dictionary-id-{nbytes}", fr.finish()[0], UNSUPPORTED))
    return bad


@pytest.fixture(scope="module")
def corpus():
    return valid_corpus()


@pytest.fixture(scope="module")
def emu():
    E = H.cuemu_library()
    vp, u32, u64 = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64
    E.emu_zstd_decode.restype = ctypes.c_int64; E.emu_zstd_decode.argtypes = [vp, u64, vp, u64]
    E.emu_zstd_decode_jump.restype = ctypes.c_int64; E.emu_zstd_decode_jump.argtypes = [vp, u64, vp, u64, u32, vp]
    E.emu_set_jump_seglog.argtypes = [u32]; E.emu_set_jump_seglog.restype = None
    return E


def emu_decode(E, comp, cap, mode=None):
    src = np.frombuffer(comp + bytes(64), dtype=np.uint8); dst = np.zeros(cap + 64, dtype=np.uint8)
    if mode is None:
        r = E.emu_zstd_decode(src.ctypes.data, len(comp), dst.ctypes.data, cap)
    else:
        nj = ctypes.c_uint32(0)
        r = E.emu_zstd_decode_jump(src.ctypes.data, len(comp), dst.ctypes.data, cap, mode, ctypes.byref(nj))
    return r, dst[:max(r, 0)].tobytes()


def oracle_verdict(comp, cap):
    src = H._np(comp); dst = np.empty(cap + 1, dtype=np.uint8)
    r = H.oracle().b2zo_zstd_decompress(dst.ctypes.data, cap, src.ctypes.data, len(comp))
    return ORACLE_RC.get(r, r) if r < 0 else dst[:r].tobytes()


def test_corpus_covers_the_format(corpus):
    """the corpus is what it claims: enough frames, and the features a name promises are there"""
    names = [n for n, *_ in corpus]
    assert len(names) == len(set(names)) and len(corpus) >= 90
    for tag in ("fcs1", "fcs2", "fcs4", "fcs8", "single1", "lit-raw-sf3", "lit-rle-sf1", "lit-huf-1s", "sf2", "sf3", "direct", "fse", "treeless",
                "seq-rle-rle-rle", "logs9.8.9", "logs5.5.5", "form1", "form2", "form3", "repeat-after-zero", "repeat-after-rle", "units-9", "rfc"):
        assert any(tag in n for n in names), tag


def ref_verdict(comp, n):
    """the reference's one-shot decoder, with a block of slack: without a content size it wants room for a whole block"""
    Z = H.ref(); src = H._np(comp); dst = np.empty(n + C.BLOCK_MAX + 1, dtype=np.uint8)
    r = Z.ZSTD_decompress(dst.ctypes.data, dst.size, src.ctypes.data, len(comp))
    return Z.ZSTD_getErrorName(r).decode() if Z.ZSTD_isError(r) else dst[:r].tobytes()


def test_writer_is_pinned_by_the_oracle_and_the_reference(corpus):
    for name, comp, plain, ref_ok in corpus:
        assert oracle_verdict(comp, len(plain)) == plain, name
        if H.ref_available():
            r = ref_verdict(comp, len(plain))
            assert (r == plain) == ref_ok, (name, r if isinstance(r, str) else len(r))


@pytest.mark.parametrize("mode", [None, 0, 2])
def test_emulated_kernels_decode_the_corpus(corpus, emu, mode):
    """the kernel sources compiled for the host: the execution units (mode None / 0) and stage J forced on every frame (mode 2)"""
    emu.emu_set_jump_seglog(30)
    for name, comp, plain, _ in corpus:
        assert emu_decode(emu, comp, len(plain), mode) == (len(plain), plain), (name, mode)


def test_emulated_kernels_decode_the_corpus_as_one_stream(corpus, emu):
    """every valid frame in one call, bare and behind size hints, with skippable frames of all 16 magic values in between: table
    chains and repcode history start afresh at each frame"""
    parts, hinted, plain = [], [], b""
    for k, (name, comp, p, _) in enumerate(corpus):
        parts.append(comp); hinted += [C.size_hint(comp), comp, C.skippable(bytes([k % 256]) * (k % 5), k % 16)]; plain += p
    emu.emu_set_jump_seglog(20)
    for stream in (b"".join(parts), b"".join(hinted)):
        for mode in (None, 2):
            r, out = emu_decode(emu, stream, len(plain), mode)
            assert r == len(plain) and out == plain, mode
        assert oracle_verdict(stream, len(plain)) == plain


def test_invalid_frames_get_the_oracle_verdict(emu):
    for name, comp, verdict in invalid_corpus():
        cap = 1 << 18
        assert oracle_verdict(comp, cap) == verdict, name
        for mode in (None, 2):
            r, _ = emu_decode(emu, comp, cap, mode)
            assert EMU_RC.get(r) == verdict, (name, mode, r)


def test_skippable_frames_of_every_magic(emu):
    fr = C.Frame(window_log=16, fcs_bytes=2); fr.raw(b"0123456789" * 40); comp, plain = fr.finish()
    for k in range(16):
        stream = C.skippable(b"user data " * k, k) + comp + C.skippable(b"", 15 - k)
        assert oracle_verdict(stream, len(plain)) == plain, k
        assert emu_decode(emu, stream, len(plain)) == (len(plain), plain), k
        if H.ref_available():
            assert H.ref_decompress(stream, len(plain)) == plain


def long_extra_bits_frame():
    """a 128 MiB window and sequences of offset code 27 with literal-length code 35 and match-length code 51: 58 extra bits in one
    sequence, more than the 57 a decoder's 64-bit container holds after a reload.  Each compressed block's sequence is followed by a
    small one whose extra bits are chosen so that the big one starts at every bit alignment (one of them at 7 bits into a byte)"""
    rng = np.random.default_rng(58)
    fr = C.Frame(window_log=27, window_mantissa=2, fcs_bytes=8)
    head = _lits(rng, 100_000, TEXT); fr.raw(head)
    for k in range(1024):
        fr.rle(k % 251, C.BLOCK_MAX)
    seen = set()
    for ml2 in (3, 35, 43, 51, 67, 99, 131, 259, 36, 45, 55, 75):
        tail = _lits(rng, 65536 + 7, TEXT)
        off = len(fr.out) + 65536 + 7 - int(rng.integers(0, 90_000))    # reaches into the raw block at the start
        assert (off + 3).bit_length() - 1 == 27
        seqs = [(65536 + 7, off + 3, 32771 + int(rng.integers(0, 20000))), (0, 1, ml2)]
        fr.compressed(tail, seqs, modes=("fse", "fse", "fse"), logs=(5, 5, 5), rng=np.random.default_rng(1))
        left = sum(nb for _, nb in fr.seq_fields[3:])                   # bits after the initial states: where the big sequence starts
        seen.add((-left) % 8)
    assert 7 in seen, seen
    return fr.finish()


@pytest.mark.parametrize("mode", [None, 2])
def test_emulated_kernels_read_58_extra_bits(emu, mode):
    """through the execution units and through stage J (in 64 MiB segments)"""
    comp, plain = long_extra_bits_frame()
    assert oracle_verdict(comp, len(plain)) == plain
    emu.emu_set_jump_seglog(26)
    assert emu_decode(emu, comp, len(plain), mode) == (len(plain), plain)


@pytest.mark.parametrize("wl", range(10, 18))
def test_small_window_frames_of_our_encoder_decode(pkg, emu, wl):
    """a window_log below 17 limits the encoder's match distances, but its blocks stay 128 KiB: the window it declares must cover a
    whole block (Block_Maximum_Size), or every decoder that follows RFC 8878 -- the reference, the oracle, the kernels -- refuses it"""
    data = pkg.corpus.g2(300_000).tobytes() + bytes(70_000)
    comp = H.oracle_compress(data, windowLog=wl)
    f0 = comp.index(struct.pack("<I", C.MAGIC))                      # (after the size hint)
    assert 10 + (comp[f0 + 5] >> 3) == 17                             # min(frame, 128 KiB) rounded up to a power of two
    assert oracle_verdict(comp, len(data)) == data
    assert emu_decode(emu, comp, len(data)) == (len(data), data)
    if H.ref_available():
        assert ref_verdict(comp, len(data)) == data


class _ZSeq(ctypes.Structure):          # ZSTD_Sequence (the reference's zstd.h)
    _fields_ = [("offset", ctypes.c_uint), ("litLength", ctypes.c_uint), ("matchLength", ctypes.c_uint), ("rep", ctypes.c_uint)]


def ref_encoder_mode_frames(pkg, corpus):
    """[(name, frame, plaintext)] written by the reference encoder in modes the rest of the suite does not use: super-blocks
    (ZSTD_c_targetCBlockSize: sub-blocks that reuse the literal and sequence tables of the sub-block before -- treeless literals,
    repeat mode), forced and disabled literal compression (ZSTD_c_literalCompressionMode), and ZSTD_compressSequences fed with the
    crafted corpus' own sequences.  Needs oracle/_ref."""
    Z = H.ref()
    Z.ZSTD_compressSequences.restype = ctypes.c_size_t
    Z.ZSTD_compressSequences.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t]
    data = pkg.corpus.g2(400_000).tobytes() + pkg.corpus.entropy_class(2, 100_000).tobytes() + bytes(30_000) + pkg.corpus.g2(70_000).tobytes()
    out = []

    def run(name, plain, params, seqs=None):
        c = Z.ZSTD_createCCtx()
        for k, v in params:
            assert not Z.ZSTD_isError(Z.ZSTD_CCtx_setParameter(c, k, v)), (name, k, v)
        src = H._np(plain); dst = np.empty(Z.ZSTD_compressBound(len(plain)) + 1024, dtype=np.uint8)
        if seqs is None:
            r = Z.ZSTD_compress2(c, dst.ctypes.data, dst.size, src.ctypes.data, len(plain))
        else:
            arr = (_ZSeq * max(len(seqs), 1))(*[_ZSeq(o, ll, ml, 0) for ll, o, ml in seqs])
            r = Z.ZSTD_compressSequences(c, dst.ctypes.data, dst.size, arr, len(seqs), src.ctypes.data, len(plain))
        Z.ZSTD_freeCCtx(c)
        assert not Z.ZSTD_isError(r), (name, Z.ZSTD_getErrorName(r))
        out.append((name, dst[:r].tobytes(), plain))

    for level in (3, 19):
        for target in (1340, 5000):
            run(f"super-blocks-L{level}-t{target}", data, [(100, level), (130, target), (201, level == 19)])
    for level in (1, 12):
        for mode in (1, 2):
            run(f"literal-mode{mode}-L{level}", data, [(100, level), (1002, mode)])
    for name, comp, plain, _ in corpus:
        fr_seqs = _corpus_sequences(name)
        if fr_seqs and len(plain) < 400_000:
            run(f"sequences-of-{name}", plain, [(100, 3), (101, 24), (1008, 0)], fr_seqs)
    return out


_SEQS = {}


def _corpus_sequences(name):
    """the (literal length, offset, match length) list of a crafted frame, over its whole plaintext"""
    if not _SEQS:
        for fname, fr in _frames_with_sequences():
            _SEQS[fname] = fr.plain_seqs
    return _SEQS.get(name)


def _frames_with_sequences():
    """a few crafted frames again, keeping the writer objects: repcode-heavy, several units, random mixtures"""
    out = []
    rng = np.random.default_rng(99)
    for i in range(6):
        fr = C.Frame(window_log=20, fcs_bytes=4)
        fr.raw(_lits(rng, 2000, TEXT))
        for b in range(1 + i % 4):
            lits = _lits(rng, 3000, TEXT)
            fr.compressed(lits, _seqs(rng, fr, 3000, 150, ml_max=200, rep=0.6), modes=("fse", "fse", "fse"), logs=(9, 8, 9), rng=rng)
        out.append((f"seqsrc-{i}", fr))
    return out


@pytest.fixture(scope="module")
def ref_mode_frames(pkg, corpus):
    if not H.ref_available():
        pytest.skip("oracle/_ref not built")
    extra = [(n, *fr.finish(), True) for n, fr in _frames_with_sequences()]
    return ref_encoder_mode_frames(pkg, corpus + extra)


def test_reference_encoder_modes_decode(ref_mode_frames, emu):
    names = [n for n, *_ in ref_mode_frames]
    assert sum(n.startswith("sequences-of-") for n in names) == 6 and any(n.startswith("super-blocks") for n in names)
    for name, comp, plain in ref_mode_frames:
        assert oracle_verdict(comp, len(plain)) == plain, name
        for mode in (None, 2):
            assert emu_decode(emu, comp, len(plain), mode) == (len(plain), plain), (name, mode)


def test_window_above_1gib_is_unsupported(emu):
    """the kernels cover windows up to 1 GiB - 16: a larger one with no content size to cut it down is refused as unsupported
    (the oracle keeps the whole output and decodes it)"""
    fr = C.Frame(window_log=30, window_mantissa=1, fcs_bytes=0); fr.raw(b"abc"); comp, plain = fr.finish()
    assert oracle_verdict(comp, 100) == plain
    assert emu_decode(emu, comp, 100)[0] == -2
