"""CPU: stage E of the Zstandard encoder (csrc/zstd_enc_entropy.cu) on mixed groups of blocks sized around E2's group of
ENT_CHAIN_BLOCKS = 16 blocks per warp, one block per lane: 15, 16, 17, 31, 32, 33 and 65 blocks.  One warp's group holds the blocks
E1 finishes itself (an RLE block, a block without sequences, a block over the body cap) beside a one-sequence block and a
32 768-sequence block, and 17, 33 and 65 leave a last group of one ragged block.  The kernel sources compiled for the host
(tests/cuemu) must write the oracle's blocks (b2zo_zstd_encode_block) byte for byte, every block must carry the decision it is
built for, and the frames must decode to the input through the emulated GPU decoder."""
import ctypes

import numpy as np
import pytest

import helpers as H
import zstd_seqsets as S

GROUP = 16                                                      # ENT_CHAIN_BLOCKS
SIZES = (15, 16, 17, 31, 32, 33, 65)
_CACHE = None


def group_cases():
    global _CACHE
    if _CACHE is None:
        rng = np.random.default_rng(16)
        _CACHE = [S.mixed_case(rng, f"chain-group-{n}-blocks", n).build() for n in SIZES]
    return _CACHE


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


def test_groups_straddle_the_chain_group_and_mix_every_kind():
    cs = group_cases()
    assert [len(c.blocks) for c in cs] == list(SIZES)
    assert {n % GROUP for n in SIZES} == {GROUP - 1, 0, 1}       # a group short by one, whole groups, a last group of one
    first = cs[SIZES.index(32)].blocks[:GROUP]                  # one warp's group of E2
    nseq = [len(sq) for sq, _ in first]
    expect = cs[SIZES.index(32)].expect
    assert 0 in nseq and 1 in nseq and S.MAXSEQ in nseq
    assert any(expect.get(b, {}).get("btype") == "rle" for b in range(GROUP))                          # finished by E1: RLE block
    assert any(expect.get(b, {}).get("btype") == "raw" and nseq[b] == S.MAXSEQ for b in range(GROUP))  # finished by E1: body cap


@pytest.mark.parametrize("n", SIZES)
def test_emulated_stage_e_on_chain_groups(emu, n):
    case = group_cases()[SIZES.index(n)]
    got = emulated_blocks(emu, case)
    S.check_branches(case, got)
    assert got == S.oracle_blocks(case), case.name
    comp = np.frombuffer(S.assemble(case, got) + bytes(64), dtype=np.uint8)
    dst = np.zeros(case.n + 64, dtype=np.uint8)
    assert emu.emu_zstd_decode(comp.ctypes.data, comp.size - 64, dst.ctypes.data, case.n) == case.n, case.name
    assert dst[:case.n].tobytes() == case.src, case.name
