"""CPU: the edges of the decoder's backward bit reader (FastBwd in csrc/zstd_dec.cu), on frames built with tests/zstd_craft.py and
decoded by the kernel sources compiled for the host (tests/cuemu), against the oracle decoder's bytes or verdict.

The reader builds its 64-bit window from aligned 8-byte words of the source and keeps the next words below it in flight, so what
can go wrong depends on where a stream lies relative to the words: the corpus puts Huffman streams (one and four per section) and
sequence bitstreams at every offset mod 8 (a skippable frame of 8 + k bytes in front), in the first words of the source (no
prefix: the words below index 0 must not be read), and ends sequence bitstreams on the source's last byte (no checksum after
the last block).  Stream sizes run from 1 byte to past the window (64 bytes) and the words in flight; the bytes directly below a
stream (its section's header, table description or jump table) are not zero and must read as zero.  Literal counts and sequence
counts one off what a stream holds make the reader run past the stream's start or leave bits unread: both are corrupt.
"""
import numpy as np
import pytest

import zstd_craft as C
from test_zstd_crafted import CORRUPT, EMU_RC, TEXT, _lits, _seqs, emu, emu_decode, oracle_verdict  # noqa: F401 (emu: fixture)

HUF_SIZES = set(range(1, 25)) | {31, 32, 33, 63, 64, 65, 66}      # the sizes (bytes) some 1-stream Huffman stream must have


def _prefix(k):
    """k in 0..7: a skippable frame of 8 + k bytes (stream offsets shift by k mod 8); 8: none"""
    return b"" if k == 8 else C.skippable(b"\xa5" * k)


def _huf_for(rng, lits, mb):
    """a Huffman table over the literals' symbols (padded to at least two) whose longest code is at most mb bits"""
    syms = sorted(set(lits))
    if len(syms) < 2:
        syms.append(syms[0] ^ 1)
    mb = max(min(mb, len(syms) - 1), (len(syms) - 1).bit_length())
    return C.Huffman(dict(zip(syms, C.huf_lengths(rng, len(syms), mb))))


def reader_corpus():
    """[(name, stream)]: valid frames and frames whose streams are read one symbol too far or too short"""
    rng = np.random.default_rng(20261017)
    out, huf_sizes = [], set()
    # ---- 1-stream Huffman literals: every stream size of HUF_SIZES at some offset mod 8 (or at the buffer's start)
    for n, alpha in [(n, a) for n in range(1, 700) for a in (TEXT[:2 + n % 7], TEXT)]:
        k = (n + len(alpha)) % 9
        lits = _lits(rng, n, alpha)
        h = _huf_for(rng, lits, 11 if n % 3 == 0 else 7)
        size = len(h.stream(lits))
        if size in huf_sizes and n > 40:
            continue
        huf_sizes.add(size)
        fr = C.Frame(window_log=17, fcs_bytes=0)
        fr.compressed(lits, _seqs(rng, fr, n, 3), lit_mode="huf", huf=h, huf_direct=True, streams=1)
        out.append((f"huf1-n{n}-a{len(alpha)}-k{k}", _prefix(k) + fr.finish()[0]))
        for d in (-1, 1):                                   # one literal fewer (bits left) or more (read below the start)
            fr = C.Frame(window_log=17, fcs_bytes=0)
            fr.compressed(lits, [], lit_mode="huf", huf=h, huf_direct=True, streams=1, lit_regen=n + d, check=False)
            out.append((f"huf1-n{n}-a{len(alpha)}-regen{d:+d}-k{k}", _prefix(k) + fr.finish()[0]))
    missing = HUF_SIZES - huf_sizes
    assert not missing, f"no 1-stream Huffman stream of {sorted(missing)} bytes"
    # ---- 4-stream Huffman literals: the jump table puts streams 2..4 at every offset
    for n in (6, 7, 9, 13, 40, 90, 250, 600, 1500):
        for k in range(9):
            lits = _lits(rng, n, TEXT if k % 2 else TEXT[:6])
            h = _huf_for(rng, lits, 11 if k % 3 == 0 else 8)
            fr = C.Frame(window_log=17, fcs_bytes=0)
            fr.compressed(lits, _seqs(rng, fr, n, 4), lit_mode="huf", huf=h, huf_direct=True, streams=4, lit_sf=1 if n < 1000 else 2)
            out.append((f"huf4-n{n}-k{k}", _prefix(k) + fr.finish()[0]))
        fr = C.Frame(window_log=17, fcs_bytes=0)
        fr.compressed(lits, [], lit_mode="huf", huf=h, huf_direct=True, streams=4, lit_sf=1 if n < 1000 else 2, lit_regen=n + 4, check=False)
        out.append((f"huf4-n{n}-regen+4", fr.finish()[0]))
    # ---- sequence bitstreams: 1 .. 60 sequences, the last block's stream ending on the source's last byte
    for nseq in list(range(1, 25)) + [28, 31, 36, 45, 60]:
        k = nseq % 9
        modes = ("pre", "pre", "pre") if nseq % 2 else ("fse", "fse", "fse")
        fr = C.Frame(window_log=16, fcs_bytes=0, checksum=nseq % 4 == 0)
        nl = 4 * nseq
        fr.compressed(_lits(rng, nl, TEXT), _seqs(rng, fr, nl, nseq, ml_max=30), lit_mode="raw", modes=modes, logs=(6, 5, 6), rng=rng)
        if nseq % 3 == 0:
            fr.compressed(_lits(rng, 20, TEXT), _seqs(rng, fr, 20, nseq, ml_max=30), lit_mode="raw", modes=("pre", "pre", "pre"))
        out.append((f"seq-n{nseq}-{modes[0]}-k{k}", _prefix(k) + fr.finish()[0]))
    # one sequence more or fewer than the stream holds: Number_of_Sequences (one byte, after the 1-byte raw literals header) patched
    for nseq in (1, 2, 5, 9, 17, 40):
        for d in (-1, 1):
            if nseq + d < 1:
                continue
            fr = C.Frame(window_log=16, fcs_bytes=0)
            nl = 20
            seqs = _seqs(rng, fr, nl, nseq, ml_max=20)
            fr.compressed(_lits(rng, nl, TEXT), seqs, lit_mode="raw", modes=("pre", "pre", "pre"))
            b = bytearray(fr.finish()[0])
            pos = len(fr.header()) + 3 + 1 + nl
            assert b[pos] == len(seqs) < 127
            b[pos] += d
            out.append((f"seq-n{nseq}-nbseq{d:+d}", bytes(b)))
    return out


@pytest.fixture(scope="module")
def corpus():
    return reader_corpus()


def test_corpus_covers_the_reader_edges(corpus):
    names = [n for n, _ in corpus]
    assert len(names) == len(set(names))
    for k in range(9):
        for kind in ("huf1-", "huf4-", "seq-"):
            assert any(n.startswith(kind) and n.endswith(f"-k{k}") for n in names), (kind, k)
    verdicts = [oracle_verdict(s, 1 << 18) for _, s in corpus]
    assert sum(v == CORRUPT for v in verdicts) >= 40 and sum(isinstance(v, bytes) for v in verdicts) >= 150


@pytest.mark.parametrize("mode", [None, 2])
def test_emulated_reader_edges_match_the_oracle(corpus, emu, mode):
    """execution units (None) and stage J (2) both take D1's output"""
    emu.emu_set_jump_seglog(30)
    for name, stream in corpus:
        want = oracle_verdict(stream, 1 << 18)
        r, got = emu_decode(emu, stream, 1 << 18, mode)
        if isinstance(want, bytes):
            assert (r, got) == (len(want), want), (name, mode, r)
        else:
            assert EMU_RC.get(r) == want, (name, mode, r, want)
