"""GPU: the hand-built LZMA2 corpus of tests/test_lzma2_crafted.py through Codec.lzma2_decompress (literal model placement chosen by
block count, in shared memory, in global memory) and the device-pointer entry point, the decoder's error codes on the invalid
streams, every valid block side by side in one launch, 3 000 blocks (more than the walk's first capacity), a 3.25 GiB block whose
matches reach distance slots 52..63 followed by a block that takes the output offsets past 2^32, a single block of 4 GiB or more
(unsupported), and the joined corpus in an .xz container."""
import ctypes
import lzma
import time
import zlib

import numpy as np
import pytest

import helpers as H
import lzma2_craft as C
from test_lzma2_crafted import (CONTEXTS, TEXT, _random_packets, _text, far_block, fill_to, header_only_stream, invalid_corpus,
                                valid_corpus)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def corpus():
    return valid_corpus()


def _device(data):
    import torch
    return torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda()


def _decode_device(c, comp, prop, cap):
    import torch
    src = _device(comp)
    dst = torch.empty(cap + 64, dtype=torch.uint8, device="cuda")
    n = c.lzma2_decompress_device(src.data_ptr(), src.numel(), prop, dst.data_ptr(), dst.numel())
    return bytes(dst[:n].cpu().numpy())


@pytest.mark.parametrize("model", [0, 1, 2])
def test_corpus_decodes(pkg, corpus, model):
    c = pkg.Codec(0, lzma2_model=model)
    try:
        for name, comp, plain, prop, _ in corpus:
            assert c.lzma2_decompress(comp, prop, max_size=len(plain)) == plain, (name, model)
            assert _decode_device(c, comp, prop, len(plain)) == plain, (name, model)
    finally:
        c.close()


def test_invalid_streams_return_corrupt(pkg):
    c = pkg.Codec(0)
    try:
        for name, comp, prop, _ in invalid_corpus():
            for call in (lambda: c.lzma2_decompress(comp, prop, max_size=1 << 22), lambda: _decode_device(c, comp, prop, 1 << 22)):
                with pytest.raises(pkg.B200zError) as e:
                    call()
                assert e.value.code == -5, (name, e.value)
    finally:
        c.close()


def joined_corpus(corpus):
    """the chunks of every valid stream, without their end markers, in one stream: each starts with a dictionary reset, so each
    stays its own block -> (stream, plaintext, dict prop, decoded offsets of the blocks)"""
    parts, plain, starts = [], b"", []
    for name, comp, p, prop, w in corpus:
        if w is None:
            continue
        starts += [len(plain) + d for _, d in w.blocks]
        parts.append(comp[:-1]); plain += p
    return b"".join(parts) + b"\x00", plain, max(prop for *_, prop, _ in corpus), starts


@pytest.mark.parametrize("model", [0, 1, 2])
def test_all_blocks_in_one_stream(pkg, corpus, model):
    """blocks of every lc + lp side by side in one launch: the literal model is sized by the largest, its stride is the GLIT one"""
    comp, plain, prop, starts = joined_corpus(corpus)
    assert len(starts) > 150
    c = pkg.Codec(0, lzma2_model=model)
    try:
        assert c.lzma2_stream_info(comp) == (len(plain), len(starts), len(comp))
        assert c.lzma2_decompress(comp, prop, max_size=len(plain)) == plain
        assert _decode_device(c, comp, prop, len(plain)) == plain
    finally:
        c.close()


def many_blocks_stream(n=3000):
    rng = np.random.default_rng(3000)
    w = C.Writer(16)
    for b in range(n):
        if b % 3 == 0:
            w.raw_chunk(_text(rng, int(rng.integers(1, 40))), True)
        else:
            w.lzma_chunk(0xE0, CONTEXTS[int(rng.integers(len(CONTEXTS)))])
            w.literals(TEXT[:int(rng.integers(1, 12))])
            _random_packets(w, rng, int(rng.integers(0, 12)))
            w.end_chunk()
    return w


@pytest.mark.parametrize("model", [0, 1, 2])
def test_many_blocks(pkg, model):
    """3 000 dictionary-reset blocks in a stream of a few KB: more than the walk's first capacity (srcSize / 65536 + 1024), so it
    runs again with room for all; with model 0 also more than fit with the literal model in shared memory"""
    w = many_blocks_stream()
    comp, plain = w.finish()
    assert len(w.blocks) == 3000 > len(comp) // 65536 + 1024
    assert H.oracle_lzma2_decompress(comp, len(plain), w.dict_prop) == (plain, len(comp))
    c = pkg.Codec(0, lzma2_model=model)
    try:
        assert c.lzma2_decompress(comp, w.dict_prop, max_size=len(plain)) == plain
        assert _decode_device(c, comp, w.dict_prop, len(plain)) == plain
    finally:
        c.close()


def far_stream():
    """a block of about 3.25 GiB at dict prop 40 whose matches reach slots 52..63, then a block of about 1 GiB -> (stream, size,
    head, far matches, start and byte of the second block)"""
    rng = np.random.default_rng(63)
    w = C.Writer(40, keep_plain=False)
    w.lzma_chunk(0xE0, (0, 0, 0))
    head, far = far_block(w, rng, range(52, 64), spread=1 << 28)
    second = w.total
    w.lzma_chunk(0xE0, (0, 0, 0)); w.literal(0x5A); w.end_chunk()
    fill_to(w, 1 << 30)
    w.end_chunk()
    comp, _ = w.finish()
    return comp, w.total, head, far, second


def test_far_distances_past_4gib(pkg):
    """decoded from device memory and compared there with the output the test builds on the device (the head, the far copies, the
    runs of the byte before); the same bytes with dict prop 39 (3 GiB) are corrupt, because the slot 63 distance exceeds it"""
    import torch
    t0 = time.perf_counter()
    comp, total, head, far, second = far_stream()
    t1 = time.perf_counter()
    assert second > 3 << 30 and total > 1 << 32 and {C.dist_slot(d - 1) for _, d, _ in far} == set(range(52, 64))
    want = torch.empty(total, dtype=torch.uint8, device="cuda")
    h = _device(head)
    want[:len(head)] = h
    fill, at = head[-1], len(head)
    for p, d, n in far:
        want[at:p] = fill
        want[p:p + n] = h[p - d:p - d + n]
        fill, at = head[p - d + n - 1], p + n
    want[at:second] = fill
    want[second:] = 0x5A
    src = _device(comp)
    dst = torch.empty(total + 64, dtype=torch.uint8, device="cuda")
    c = pkg.Codec(0)
    try:
        torch.cuda.synchronize(); t2 = time.perf_counter()
        n = c.lzma2_decompress_device(src.data_ptr(), src.numel(), 40, dst.data_ptr(), dst.numel())
        torch.cuda.synchronize(); t3 = time.perf_counter()
        assert n == total and torch.equal(dst[:n], want)
        with pytest.raises(pkg.B200zError) as e:
            c.lzma2_decompress_device(src.data_ptr(), src.numel(), 39, dst.data_ptr(), dst.numel())
        assert e.value.code == -5
    finally:
        c.close()
    print(f"far distances: stream {len(comp) / 2**20:.2f} MiB built in {t1 - t0:.1f} s, {total / 2**30:.2f} GiB decoded in "
          f"{1e3 * (t3 - t2):.0f} ms, peak device memory {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB (torch allocations)")


def test_block_of_4gib_is_unsupported(pkg, codec):
    comp = header_only_stream()
    with pytest.raises(pkg.B200zError) as e:
        codec.lzma2_decompress(comp, 24, max_size=1 << 20)
    assert e.value.code == -6
    src = _device(comp)
    with pytest.raises(pkg.B200zError) as e:
        codec.lzma2_decompress_device(src.data_ptr(), src.numel(), 24, src.data_ptr(), 0)
    assert e.value.code == -6


def test_xz_of_the_joined_corpus(pkg, corpus, codec):
    comp, plain, prop, starts = joined_corpus(corpus)
    L = pkg.load_library()
    vp, sz, u32 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32
    L.b200z_xz_wrap_bound.restype = sz; L.b200z_xz_wrap_bound.argtypes = [sz, u32]
    L.b200z_xz_wrap.argtypes = [vp, sz, u32, u32, vp, u32, u32, u32, vp, sz, ctypes.POINTER(sz)]
    ends = starts[1:] + [len(plain)]
    checks = np.array([zlib.crc32(plain[a:b]) for a, b in zip(starts, ends)], dtype=np.uint64)
    src = np.frombuffer(comp, dtype=np.uint8)
    cap = L.b200z_xz_wrap_bound(len(comp), len(checks)); out = np.zeros(cap, dtype=np.uint8); n = ctypes.c_size_t()
    assert L.b200z_xz_wrap(src.ctypes.data, len(comp), prop, 1, checks.ctypes.data, len(checks), 0, 0, out.ctypes.data, cap, ctypes.byref(n)) == 0
    xz = out[:n.value].tobytes()
    assert lzma.decompress(xz, format=lzma.FORMAT_XZ) == plain
    assert codec.xz_decompress(xz) == plain
