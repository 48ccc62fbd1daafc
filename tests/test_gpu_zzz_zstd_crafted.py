"""GPU: the hand-built conformance corpus of tests/test_zstd_crafted.py through Codec.decompress -- the execution units, stage J
(automatic and forced, whole and in 1 MiB segments), the host pipeline in small batches and the device-pointer entry point -- plus
the decoder's error codes on the invalid frames, and every valid frame in one call (tables and repcode history start afresh at
each frame inside one launch); frames with offsets above 2^29 in a 768 MiB window, a window above 1 GiB (unsupported), the 58-extra-bit
frame, and the reference encoder's super-block, literal-compression-mode and compressSequences frames."""
import numpy as np
import pytest

import helpers as H
import zstd_craft as C
from test_zstd_crafted import (CHECKSUM, CORRUPT, UNSUPPORTED, _frames_with_sequences, invalid_corpus, long_extra_bits_frame,
                               ref_encoder_mode_frames, valid_corpus)

pytestmark = pytest.mark.gpu

ERR = {CORRUPT: -5, UNSUPPORTED: -6, CHECKSUM: -8}


@pytest.fixture(scope="module")
def corpus():
    return valid_corpus()


@pytest.mark.parametrize("params", [dict(dec_jump=0), dict(dec_jump=1), dict(dec_jump=2), dict(dec_jump=2, dec_jump_seg_log=20)])
def test_corpus_decodes(pkg, corpus, params):
    c = pkg.Codec(0, **params)
    try:
        for name, comp, plain, _ in corpus:
            assert c.decompress(comp, max_size=len(plain)) == plain, (name, params)
    finally:
        c.close()


def test_corpus_as_one_stream(pkg, corpus):
    """all valid frames in one call, bare and behind size hints with skippable frames of every magic between them; also through
    the host pipeline in small batches and from device memory"""
    import torch
    parts, hinted, plain = [], [], b""
    for k, (name, comp, p, _) in enumerate(corpus):
        parts.append(comp); hinted += [C.size_hint(comp), comp, C.skippable(bytes([k % 256]) * (k % 5), k % 16)]; plain += p
    for params in (dict(), dict(dec_jump=2)):
        c = pkg.Codec(0, **params)
        try:
            for stream in (b"".join(parts), b"".join(hinted)):
                assert c.decompress(stream, max_size=len(plain)) == plain, params
                src = torch.from_numpy(np.frombuffer(stream, dtype=np.uint8).copy()).cuda()
                dst = torch.empty(len(plain) + 64, dtype=torch.uint8, device="cuda")
                n = c.decompress_device(src.data_ptr(), src.numel(), dst.data_ptr(), dst.numel())
                assert n == len(plain) and bytes(dst[:n].cpu().numpy()) == plain, params
        finally:
            c.close()


def test_corpus_in_small_host_batches(pkg, corpus):
    """the host pipeline cuts a stream into batches of whole frames by their declared sizes: the frames that declare one, three
    times over (about 13 MiB), in 4 MiB batches"""
    sized = [(comp, p) for _, comp, p, _ in corpus if (comp[4] >> 6) or (comp[4] >> 5) & 1]
    stream = b"".join(comp for comp, _ in sized) * 3; plain = b"".join(p for _, p in sized) * 3
    c = pkg.Codec(0, host_batch_log=22)
    try:
        assert c.decompress(stream, max_size=len(plain)) == plain
    finally:
        c.close()


@pytest.mark.parametrize("dec_jump", [0, 2])
def test_invalid_frames_return_the_error_code(pkg, dec_jump):
    """-5 corrupt, -6 unsupported, -8 checksum: the verdicts the oracle gives these frames (tests/test_zstd_crafted.py)"""
    c = pkg.Codec(0, dec_jump=dec_jump)
    try:
        for name, comp, verdict in invalid_corpus():
            with pytest.raises(Exception) as e:
                c.decompress(comp, max_size=1 << 18)
            assert getattr(e.value, "code", None) == ERR[verdict], (name, e.value)
    finally:
        c.close()


@pytest.mark.parametrize("dec_jump", [0, 2])
def test_58_extra_bits(pkg, dec_jump):
    comp, plain = long_extra_bits_frame()
    c = pkg.Codec(0, dec_jump=dec_jump)
    try:
        assert c.decompress(comp, max_size=len(plain)) == plain
    finally:
        c.close()


def test_window_above_1gib_returns_unsupported(pkg, codec):
    fr = C.Frame(window_log=30, window_mantissa=1, fcs_bytes=0); fr.raw(b"abc")
    with pytest.raises(Exception) as e:
        codec.decompress(fr.finish()[0], max_size=100)
    assert getattr(e.value, "code", None) == -6


def test_reference_encoder_modes(pkg, corpus):
    if not H.ref_available():
        pytest.skip("oracle/_ref not built")
    extra = [(n, *fr.finish(), True) for n, fr in _frames_with_sequences()]
    frames = ref_encoder_mode_frames(pkg, corpus + extra)
    for dec_jump in (0, 2):
        c = pkg.Codec(0, dec_jump=dec_jump)
        try:
            for name, comp, plain in frames:
                assert c.decompress(comp, max_size=len(plain)) == plain, (name, dec_jump)
        finally:
            c.close()


def test_large_offsets(pkg):
    """a window of 768 MiB and 700 MiB of raw blocks, then compressed blocks whose sequences copy from more than 2^29 bytes back
    (offset code 29) with the largest literal-length and match-length codes (60 extra bits): decoded from device memory by the
    execution units and by stage J (whole and in 256 MiB segments), compared on the device"""
    import time
    import torch
    rng = np.random.default_rng(29)
    head = rng.integers(0, 256, size=700 << 20, dtype=np.uint8)
    fr = C.Frame(window_log=29, window_mantissa=4, fcs_bytes=8)
    fr.out = bytearray(head.tobytes()); fr._pending = len(fr.out)         # the raw blocks, written below with numpy
    for ml2 in (3, 35, 43, 51, 67, 99, 131, 259):
        tail = rng.integers(0, 256, size=65536 + 9, dtype=np.uint8).tobytes()
        off = len(fr.out) + 65536 + 9 - int(rng.integers(1, 100_000))    # into the first 100 KB of the frame
        assert (off + 3).bit_length() - 1 == 29 and off > (1 << 29)
        fr.compressed(tail, [(65536 + 9, off + 3, 32771 + int(rng.integers(0, 30000))), (0, 1, ml2)], modes=("fse",) * 3, logs=(5, 5, 5),
                      rng=np.random.default_rng(1))
    plain = bytes(fr.out)
    hdr = fr.header()
    nraw = len(head) // C.BLOCK_MAX
    bh = (np.uint32(C.BLOCK_MAX) << 3).astype("<u4").tobytes()[:3]         # raw, not last
    raw = np.concatenate([np.frombuffer(bh * nraw, dtype=np.uint8).reshape(nraw, 3), head.reshape(nraw, C.BLOCK_MAX)], axis=1).ravel()
    fr.blocks[-1][3] = True
    rest = b"".join((int(last) | (t << 1) | (n << 3)).to_bytes(3, "little") + body for t, n, body, last in fr.blocks)
    comp = np.concatenate([np.frombuffer(hdr, dtype=np.uint8), raw, np.frombuffer(rest, dtype=np.uint8)])
    src = torch.from_numpy(comp).cuda()
    want = torch.from_numpy(np.frombuffer(plain, dtype=np.uint8).copy()).cuda()
    del head, raw, comp
    dst = torch.empty(len(plain) + 64, dtype=torch.uint8, device="cuda")
    for params in (dict(dec_jump=0), dict(dec_jump=2), dict(dec_jump=2, dec_jump_seg_log=28)):
        c = pkg.Codec(0, **params)
        try:
            free0 = torch.cuda.mem_get_info()[0]
            torch.cuda.synchronize(); t0 = time.perf_counter()
            n = c.decompress_device(src.data_ptr(), src.numel(), dst.data_ptr(), dst.numel())
            torch.cuda.synchronize(); t1 = time.perf_counter()
            used = free0 - torch.cuda.mem_get_info()[0]                   # the codec's scratch, which it keeps after the call
            print(f"large offsets {params}: {len(plain) / 2**20:.0f} MiB in {1e3 * (t1 - t0):.1f} ms, decoder scratch {used / 2**20:.0f} MiB")
            assert n == len(plain) and torch.equal(dst[:n], want), params
        finally:
            c.close()


@pytest.mark.parametrize("wl", [10, 12, 16, 17])
def test_small_window_round_trip(pkg, wl):
    """window_log below 17: the encoder's matches stay within the window, its blocks stay 128 KiB, and the window it declares covers a
    whole block -- the same bytes as the oracle, restored by the GPU decoder (and by the reference where built)"""
    data = pkg.corpus.g2(900_000).tobytes()
    c = pkg.Codec(0, window_log=wl)
    try:
        comp = c.compress(data)
        assert comp == H.oracle_compress(data, windowLog=wl)
        assert c.decompress(comp) == data
    finally:
        c.close()
    if H.ref_available():
        assert H.ref_decompress(comp, len(data)) == data
