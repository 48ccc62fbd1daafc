"""Tables taken from an earlier block that another CTA decodes.

Treeless literals and repeat-mode sequence tables reuse the tables of the last block that defined them.  The decoder's entropy
stage builds every block's tables in the shared memory of the CTA that decodes the block (csrc/zstd_dec.cu, zstd_dec_lit_streams_kernel:
B2Z_LIT_BLOCKS blocks per CTA, zstd_dec_seq_streams_kernel: groups of B2Z_SEQ_BLOCKS), so the defining block may belong to another CTA's group.
These frames put it k blocks back, for k from 1 to past the larger group, with raw, RLE and compressed blocks (raw / RLE
literals, no sequences) in between and a varying number of raw blocks in front, so that the two blocks fall at every offset
within and across the groups.  The emulated kernels (CPU) and the codec (GPU) must give the oracle's bytes.
"""
import ctypes

import numpy as np
import pytest

import helpers as H
import zstd_craft as C
from test_zstd_crafted import TEXT, _huf, _lits, _seqs

LIT_BLOCKS, SEQ_BLOCKS = 16, 17          # zstd_dec.cu: B2Z_LIT_BLOCKS, B2Z_SEQ_BLOCKS
KS = list(range(1, max(LIT_BLOCKS, SEQ_BLOCKS) + 3))


def cross_frames():
    """[(k, frame, plaintext)]: the block that defines the Huffman and FSE tables, k - 1 blocks without tables, then a block with
    treeless literals and sequences in repeat mode for all three tables"""
    rng = np.random.default_rng(20261017)
    out = []
    for k in KS:
        fr = C.Frame(window_log=17, fcs_bytes=4, checksum=bool(k & 1))
        for _ in range(k % 7):
            fr.raw(_lits(rng, int(rng.integers(1, 200)), TEXT))
        lits = _lits(rng, 3000, TEXT)
        h = _huf(rng, lits, 11, extra=TEXT)
        fr.compressed(lits, _seqs(rng, fr, 3000, 60), lit_mode="huf", huf=h, streams=4,
                      modes=("fse", "fse", "fse"), logs=(7, 6, 7), rng=rng, full=(True,) * 3)
        for i in range(k - 1):
            kind = i % 4
            if kind == 0:
                fr.raw(_lits(rng, int(rng.integers(1, 300)), TEXT))
            elif kind == 1:
                fr.rle(int(rng.integers(256)), int(rng.integers(1, 5000)))
            elif kind == 2:
                fr.compressed(_lits(rng, int(rng.integers(1, 400)), TEXT), [], lit_mode="raw")
            else:
                fr.compressed(bytes([0x20]) * int(rng.integers(1, 400)), [], lit_mode="rle")
        streams = 4 if k % 3 else 1
        tl = _lits(rng, 1500 if streams == 4 else 900, TEXT)                # (one stream: a literals size under 1 KiB)
        fr.compressed(tl, _seqs(rng, fr, len(tl), 40), lit_mode="treeless", streams=streams, modes=("rep", "rep", "rep"))
        comp, plain = fr.finish()
        out.append((k, comp, plain))
    return out


@pytest.fixture(scope="module")
def frames():
    F = cross_frames()
    for k, comp, plain in F:                                        # the writer is pinned by the oracle
        src = H._np(comp); dst = np.empty(len(plain) + 1, dtype=np.uint8)
        r = H.oracle().b2zo_zstd_decompress(dst.ctypes.data, len(plain), src.ctypes.data, len(comp))
        assert r == len(plain) and dst[:r].tobytes() == plain, k
    return F


def test_emulated_kernels_take_tables_from_other_ctas(frames):
    E = H.cuemu_library()
    E.emu_zstd_decode.restype = ctypes.c_int64
    E.emu_zstd_decode.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_uint64]
    for k, comp, plain in frames:
        src = np.frombuffer(comp + bytes(64), dtype=np.uint8); dst = np.zeros(len(plain) + 64, dtype=np.uint8)
        r = E.emu_zstd_decode(src.ctypes.data, len(comp), dst.ctypes.data, len(plain))
        assert r == len(plain) and dst[:r].tobytes() == plain, k
    stream = b"".join(c for _, c, _ in frames)                      # one batch: the frames' blocks side by side in the same groups
    plain = b"".join(p for _, _, p in frames)
    src = np.frombuffer(stream + bytes(64), dtype=np.uint8); dst = np.zeros(len(plain) + 64, dtype=np.uint8)
    r = E.emu_zstd_decode(src.ctypes.data, len(stream), dst.ctypes.data, len(plain))
    assert r == len(plain) and dst[:r].tobytes() == plain


@pytest.mark.gpu
def test_gpu_takes_tables_from_other_ctas(frames, pkg):
    c = pkg.Codec(0)
    for k, comp, plain in frames:
        assert c.decompress(comp, len(plain)) == plain, k
    stream = b"".join(cm for _, cm, _ in frames)
    plain = b"".join(p for _, _, p in frames)
    assert c.decompress(stream, len(plain)) == plain
    c.close()
