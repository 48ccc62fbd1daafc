"""CPU: stage E of the Zstandard encoder (csrc/zstd_enc_entropy.cu, the entropy coder) on the hand-built sequence sets of
tests/zstd_seqsets.py, which reach the branches the parses rarely produce -- every literals form and header size, deep Huffman
trees, both Huffman descriptions, every sequence-count form and table mode, every length code, offset codes up to 27, the RLE
block and its near misses, the raw fallbacks and groups of blocks of mixed kinds.

For every case the kernel sources compiled for the host (tests/cuemu) must write the oracle's blocks byte for byte
(b2zo_zstd_encode_block), every block must carry the decision its case is named for, and the blocks, put into the encoder's
frames, must decode to the input through the oracle decoder, the emulated GPU decoder and, where oracle/_ref is built, the
reference decoder -- the one judge here that shares nothing with the encoder."""
import ctypes

import numpy as np
import pytest

import helpers as H
import zstd_seqsets as S


@pytest.fixture(scope="module")
def emu():
    E = H.cuemu_library()
    vp, u32, u64 = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64
    E.emu_zstd_enc_entropy.restype = u64; E.emu_zstd_enc_entropy.argtypes = [vp, u64, u32, u32, vp, vp, vp, vp, vp, vp, u32]
    E.emu_slot_bytes.restype = u32
    E.emu_zstd_decode.restype = ctypes.c_int64; E.emu_zstd_decode.argtypes = [vp, u64, vp, u64]
    return E


def emulated_blocks(E, case):
    src, seqs, nseq, lits, nlit = case.arrays()
    nb, SLOT = len(case.blocks), E.emu_slot_bytes()
    slots = np.full(nb * SLOT, 0xCD, dtype=np.uint8); ssz = np.zeros(nb, dtype=np.uint32)
    E.emu_zstd_enc_entropy(src.ctypes.data, case.n, case.frame_log, 1, seqs.ctypes.data, nseq.ctypes.data, lits.ctypes.data,
                           nlit.ctypes.data, slots.ctypes.data, ssz.ctypes.data, nb)
    return [slots[b * SLOT:b * SLOT + ssz[b]].tobytes() for b in range(nb)]


def test_sets_cover_what_they_claim():
    cs = S.cases()
    names = [c.name for c in cs]
    for tag in ("lit-raw-0", "lit-rle-4096", "lit-huf-257", "lit-huf-16384", "huf-deep-several-halvings", "huf-over-128-weights-fse",
                "nbseq-32512", "nbseq-32768", "mode-rle-of", "table-largest-logs", "ll-every-code", "ml-every-code",
                "offset-codes-to-27-parity", "wide-sequence-parity", "body-cap-raw", "group-31-blocks"):
        assert tag in names, tag
    assert sorted(len(c.blocks) for c in cs if c.name.startswith("group-")) == [9, 10, 11, 29, 31]
    assert all(c.expect for c in cs)


@pytest.mark.parametrize("name", [c.name for c in S.cases()])
def test_oracle_blocks_take_the_named_branch_and_decode(name):
    case = next(c for c in S.cases() if c.name == name)
    blocks = S.oracle_blocks(case)
    S.check_branches(case, blocks)
    if case.parity_only:
        return
    comp = S.assemble(case, blocks)
    assert H.oracle_decompress(comp, case.n) == case.src
    if H.ref_available():
        assert H.ref_decompress(comp, case.n) == case.src


def test_emulated_stage_e_writes_the_oracle_blocks(emu):
    for case in S.cases():
        assert emulated_blocks(emu, case) == S.oracle_blocks(case), case.name


def test_emulated_stage_e_on_all_sets_in_few_launches(emu):
    """the cases back to back, one input per frame log: blocks of every kind side by side in E2's groups of ten"""
    for case in S.launches(S.cases()):
        got = emulated_blocks(emu, case)
        S.check_branches(case, got)
        assert got == S.oracle_blocks(case), case.name
        if not case.parity_only:
            comp = np.frombuffer(S.assemble(case, got) + bytes(64), dtype=np.uint8)
            dst = np.zeros(case.n + 64, dtype=np.uint8)
            assert emu.emu_zstd_decode(comp.ctypes.data, comp.size - 64, dst.ctypes.data, case.n) == case.n, case.name
            assert dst[:case.n].tobytes() == case.src, case.name
