"""GPU: stage E of the Zstandard encoder (the E1 / E2 / E3 kernels of csrc/zstd_enc_entropy.cu) through Codec.stage_e on the mixed
groups of tests/test_zstd_enc_entropy_groups.py, sized around E2's group of 16 blocks per warp (15, 16, 17, 31, 32, 33 and 65
blocks; one warp's group holds an RLE block, a block without sequences and a block over the body cap beside one-sequence and
32 768-sequence blocks).  The blocks must be the oracle's (b2zo_zstd_encode_block) byte for byte, carry the decision they are built
for, and decode through Codec.decompress and, where oracle/_ref is built, the reference decoder."""
import pytest

import helpers as H
import zstd_seqsets as S
from test_zstd_enc_entropy_groups import SIZES, group_cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def codec(pkg):
    c = pkg.Codec(0, frame_log=group_cases()[0].frame_log)
    yield c
    c.close()


@pytest.mark.parametrize("n", SIZES)
def test_stage_e_on_chain_groups(codec, n):
    case = group_cases()[SIZES.index(n)]
    src, seqs, nseq, lits, nlit = case.arrays()
    data, sizes = codec.stage_e(src[:case.n], seqs, nseq, lits, nlit)
    got = S.split_blocks(data, sizes)
    assert got == S.oracle_blocks(case), case.name
    S.check_branches(case, got)
    comp = S.assemble(case, got)
    assert codec.decompress(comp, max_size=case.n) == case.src, case.name
    if H.ref_available():
        assert H.ref_decompress(comp, case.n) == case.src, case.name
