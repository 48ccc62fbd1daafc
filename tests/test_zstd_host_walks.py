"""CPU: the host's walks over zstd frame and block headers -- b200z_zstd_frame_info (what a whole stream decodes to) and
b200z_zstd_frame_prefix (the complete frames at the start of a buffer, for readers that take a packed stream piece by piece) -- on
the hand-built frames of tests/test_zstd_crafted.py: one by one, joined into one stream behind size hints with skippable frames
in between, cut at every frame boundary and at seeded points, and followed by the header faults the decoder refuses."""
import ctypes

import numpy as np
import pytest

import helpers as H
import zstd_craft as C
from test_zstd_crafted import invalid_corpus, valid_corpus

OK, CORRUPT, UNSUPPORTED = 0, -5, -6
HEADER_FAULTS = ("block-type-reserved", "frame-header-reserved-bit", "window-exponent-over-31", "raw-block-over-limit", "rle-block-over-limit",
                 "raw-block-over-window", "rle-block-over-window")


@pytest.fixture(scope="module")
def lib(pkg):
    L = pkg.load_library()
    sz, u64, u32 = ctypes.c_size_t, ctypes.c_uint64, ctypes.c_uint32
    L.b200z_zstd_frame_info.argtypes = [ctypes.c_void_p, sz, ctypes.POINTER(u64), ctypes.POINTER(u32)]
    L.b200z_zstd_frame_prefix.argtypes = [ctypes.c_void_p, sz, u64, ctypes.POINTER(sz), ctypes.POINTER(u64), ctypes.POINTER(u32)]
    return L


def frame_info(L, buf, n=None):
    cs, nf = ctypes.c_uint64(), ctypes.c_uint32()
    rc = L.b200z_zstd_frame_info(buf.ctypes.data, len(buf) if n is None else n, ctypes.byref(cs), ctypes.byref(nf))
    return rc, cs.value, nf.value


def frame_prefix(L, buf, n=None, max_content=1 << 62):
    """(rc, usedBytes, contentBound, nFrames); the outputs start as values no answer has, so one left unwritten shows"""
    used, bound, nf = ctypes.c_size_t(2**64 - 1), ctypes.c_uint64(2**64 - 1), ctypes.c_uint32(2**32 - 1)
    rc = L.b200z_zstd_frame_prefix(buf.ctypes.data, len(buf) if n is None else n, max_content, ctypes.byref(used), ctypes.byref(bound), ctypes.byref(nf))
    return rc, used.value, bound.value, nf.value


def layout(frame):
    """(declares its size, raw + RLE bytes, raw + RLE bytes + 128 KiB per compressed block) of one frame, from its headers"""
    fhd = frame[4]
    single, fcs_flag = (fhd >> 5) & 1, fhd >> 6
    p = 5 + (not single) + (0, 1, 2, 4)[fhd & 3] + ((single, 2, 4, 8)[fcs_flag])
    lower = compressed = 0
    while True:
        bh = int.from_bytes(frame[p:p + 3], "little"); p += 3
        btype, bsize = (bh >> 1) & 3, bh >> 3
        if btype == 2:
            compressed += 1
        else:
            lower += bsize
        p += 1 if btype == 1 else bsize
        if bh & 1:
            return bool(fcs_flag or single), lower, lower + C.BLOCK_MAX * compressed


@pytest.fixture(scope="module")
def frames():
    """[(frame, plaintext, declared, lower bound, upper bound)] of the valid corpus"""
    return [(comp, plain, *layout(comp)) for _, comp, plain, _ in valid_corpus()]


def joined(frames):
    """the frames in one stream behind size hints, skippable frames of every magic value in between (as
    test_emulated_kernels_decode_the_corpus_as_one_stream builds it): (stream, [(start, end, content or None for a skippable frame)])"""
    units, out = [], b""
    for k, (comp, plain, declared, _, bound) in enumerate(frames):
        for part, content in ((C.size_hint(comp), None), (comp, len(plain) if declared else bound), (C.skippable(bytes([k % 256]) * (k % 5), k % 16), None)):
            units.append((len(out), len(out) + len(part), content)); out += part
    return out, units


def expected_prefix(units, cut, max_content=1 << 62):
    """what frame_prefix reports for the first `cut` bytes: whole frames up to the first one cut off or past max_content (the first
    is always taken); a skippable frame goes with the frame before it, or with the one after when none has been taken"""
    used = bound = n = 0
    for start, end, content in units:
        if end > cut or (content is not None and n and bound + content > max_content):
            break
        if content is None:
            used = end if n else used
        else:
            used, bound, n = end, bound + content, n + 1
    return used, bound, n


def test_frame_info_on_each_frame(lib, frames):
    for comp, plain, declared, lower, _ in frames:
        got = frame_info(lib, H._np(comp))
        assert got == ((OK, len(plain), 1) if declared else (UNSUPPORTED, lower, 1)), (got, declared, lower)


def test_frame_info_on_the_joined_stream(lib, frames):
    """bare and behind size hints: the declared sizes plus the lower bounds of the frames without one"""
    stream, _ = joined(frames)
    bare = b"".join(f[0] for f in frames)
    total = sum(len(plain) if declared else lower for _, plain, declared, lower, _ in frames)
    assert not all(f[2] for f in frames)
    for s in (bare, stream):
        assert frame_info(lib, H._np(s)) == (UNSUPPORTED, total, len(frames))
    declared = [f for f in frames if f[2]]
    assert frame_info(lib, H._np(b"".join(f[0] for f in declared))) == (OK, sum(len(f[1]) for f in declared), len(declared))


def test_frame_prefix_cuts_at_frame_boundaries(lib, frames):
    """at every frame boundary +-1 and at 200 seeded cut points of the joined stream: the complete frames in front of the cut"""
    stream, units = joined(frames)
    buf = H._np(stream)
    rng = np.random.default_rng(8878)
    points = {b + e for start, end, _ in units for b in (start, end) for e in (-1, 0, 1)}
    extra = {int(x) for x in rng.integers(0, len(stream) + 1, 200)}
    assert len(extra - points) >= 190
    for cut in sorted(p for p in points | extra if 0 <= p <= len(stream)):
        assert frame_prefix(lib, buf, cut) == (OK, *expected_prefix(units, cut)), cut
    assert expected_prefix(units, len(stream)) == (len(stream), sum(u[2] for u in units if u[2] is not None), len(frames))


def test_frame_prefix_stops_at_max_content(lib, frames):
    """one byte either side of each frame's running sum: the walk stops before a frame that would take the sum past maxContent"""
    stream, units = joined(frames)
    buf = H._np(stream)
    total = 0
    for _, _, content in units:
        if content is None:
            continue
        total += content
        for mc in (total - 1, total, total + 1):
            assert frame_prefix(lib, buf, max_content=mc) == (OK, *expected_prefix(units, len(stream), mc)), mc


def damaged_frames():
    """[(name, frame)]: the header faults of invalid_corpus() that the decoder calls corrupt, and 4 bytes that are no frame"""
    bad = [(name, comp) for name, comp, _ in invalid_corpus() if name in HEADER_FAULTS]
    assert sorted(n for n, _ in bad) == sorted(HEADER_FAULTS)
    assert any(comp[5] >= 0xB0 for n, comp in bad if n == "window-exponent-over-31")
    return bad + [("junk", b"junk")]


def test_frame_prefix_delivers_the_frames_in_front_of_damage(lib, frames):
    """[valid frames][damaged frame]: corrupt, with every output describing the valid frames in front (none in front: all zero)"""
    stream, units = joined(frames[:5])
    for name, bad in damaged_frames():
        for head, head_units in ((stream, units), (b"", [])):
            got = frame_prefix(lib, H._np(head + bad))
            assert got == (CORRUPT, *expected_prefix(head_units, len(head))), (name, len(head), got)


def test_frame_info_refuses_damage(lib, frames):
    stream, _ = joined(frames[:5])
    for name, bad in damaged_frames():
        assert frame_info(lib, H._np(stream + bad))[0] == CORRUPT, name
