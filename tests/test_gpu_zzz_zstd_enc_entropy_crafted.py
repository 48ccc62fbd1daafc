"""GPU: stage E of the Zstandard encoder (the E1 / E2 / E3 kernels of csrc/zstd_enc_entropy.cu) on the hand-built sequence sets of
tests/zstd_seqsets.py through Codec.stage_e, which runs stage E alone on given sequences with its slots and scratch filled with 0xCD
first.  Every case in a launch of its own, then all of them in as few launches as their frame logs allow: the blocks must be the
oracle's (b2zo_zstd_encode_block) byte for byte and carry the decision their case is named for, and the frames must decode through
Codec.decompress and the reference decoder.  Two sets only the GPU takes: offset codes up to 26 in a valid 2^27-byte frame, and one
launch of smCount * 64 + 37 blocks, where E1 and E3 (grid capped at smCount * 16 CTAs of 4 warps) take a second lap of their
grid-stride loop over real cases."""
import numpy as np
import pytest

import helpers as H
import zstd_seqsets as S

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def codecs(pkg):
    made = {}

    def get(frame_log):
        if frame_log not in made:
            # frames above 2^24 bytes exist only in the long mode (8 windows per frame); stage E reads nothing else of it
            made[frame_log] = pkg.Codec(0, long=frame_log - 3) if frame_log > 24 else pkg.Codec(0, frame_log=frame_log)
        return made[frame_log]
    yield get
    for c in made.values():
        c.close()


def run(codec, case):
    src, seqs, nseq, lits, nlit = case.arrays()
    data, sizes = codec.stage_e(src[:case.n], seqs, nseq, lits, nlit)
    return S.split_blocks(data, sizes)


def check(codec, case, got, want=None):
    assert got == (want if want is not None else S.oracle_blocks(case)), case.name
    S.check_branches(case, got)
    if case.parity_only:
        return
    comp = S.assemble(case, got)
    assert codec.decompress(comp, max_size=case.n) == case.src, case.name
    if H.ref_available():
        assert H.ref_decompress(comp, case.n) == case.src, case.name


def test_each_case_in_its_own_launch(codecs):
    for case in S.cases():
        c = codecs(case.frame_log)
        check(c, case, run(c, case))


def test_all_cases_in_few_launches(codecs):
    for case in S.launches(S.cases()):
        c = codecs(case.frame_log)
        check(c, case, run(c, case))


def test_offset_codes_to_26_in_a_2e27_frame(codecs):
    case = S.large_offset_case()
    c = codecs(case.frame_log)
    check(c, case, run(c, case))


def test_grid_stride_second_lap(codecs):
    import torch
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    case = S.grid_case(sm)
    assert len(case.blocks) == sm * 64 + 37
    c = codecs(case.frame_log)
    got = run(c, case)
    want = S.oracle_blocks(case)
    assert all(b != case.blocks[0] for b in case.blocks[sm * 64:])  # every block of the second lap is a real case, none a zero block
    check(c, case, got, want)
