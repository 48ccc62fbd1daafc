"""GPU: the RISC-V branch converter (csrc/b2z_filter.cu riscv_*_kernel) through the C ABI and the .xz writer and reader, against the
oracle's statement and -- where oracle/_ref exists -- the reference's converter and unpacker.  The kernel sources are checked on the CPU
through the host emulation in tests/test_riscv_filter.py."""
import ctypes

import numpy as np
import pytest

import helpers as H
from test_riscv_filter import ADVERSARIAL, RISCV, call_heavy_riscv, foreign_xz, oracle_riscv, ref_riscv, riscv_soup
from test_xz_container import _lib, _parse, _ref_unpack

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def soup():
    return riscv_soup(1_500_000, 61)                                 # ~8 MB


def test_filter_equals_the_oracle_and_the_reference(pkg, codec, soup):
    late = bytearray(ADVERSARIAL * 300_000); late[300_001] = 0x13
    for data in (soup + ADVERSARIAL * 500_000 + soup[:100_001], bytes(late)):
        for pc in (0, 0x00ABC000, 0xFFFFFFFE):
            enc = codec.filter(RISCV, True, data, pc)
            assert enc == oracle_riscv(1, data, pc), hex(pc)
            assert codec.filter(RISCV, False, enc, pc) == data, hex(pc)
            dec = codec.filter(RISCV, False, data, pc)
            assert dec == oracle_riscv(0, data, pc), hex(pc)
            r = ref_riscv(1, data, pc)
            assert r is None or (r == enc and ref_riscv(0, data, pc) == dec)
    for n in range(10):
        for enc in (True, False):
            assert codec.filter(RISCV, enc, soup[:n], 0x1000) == oracle_riscv(int(enc), soup[:n], 0x1000), n
    with pytest.raises(pkg.B200zError) as e:
        codec.filter(RISCV, True, soup[:1000], 0x1001)              # odd start offset (BranchMisc.cpp:57,99; XzDec.c:124)
    assert e.value.code == -6


def test_device_buffer_of_256_mib(pkg, codec, soup):
    n = 256 << 20
    tile = np.frombuffer(soup[:(4 << 20) + 2] + ADVERSARIAL * 20_001, dtype=np.uint8)
    data = np.resize(tile, n)                                        # the tile's odd length in halfwords moves every CTA's phase
    data[n // 3] ^= 0x55
    L = codec.L
    d = ctypes.c_void_p()
    codec._check(L.b200z_dev_alloc(codec.h, ctypes.byref(d), n))
    try:
        for pc, enc in ((0x00ABC000, 1), (0x00ABC000, 0)):
            codec._check(L.b200z_dev_upload(codec.h, d, data.ctypes.data, n))
            codec._check(L.b200z_filter_device(codec.h, RISCV, enc, d, n, pc))
            got = np.empty(n, dtype=np.uint8)
            codec._check(L.b200z_dev_download(codec.h, got.ctypes.data, d, n))
            want = np.frombuffer(oracle_riscv(enc, data.tobytes(), pc), dtype=np.uint8)
            assert np.array_equal(got, want), enc
    finally:
        L.b200z_dev_free(codec.h, d)


def _block_payloads(L, xz):
    rc, blocks, _ = _parse(L, xz)
    assert rc == 0
    out = []
    for b in blocks:
        raw = xz[b.packOff:b.packOff + b.packSize]
        plain, used = H.oracle_lzma2_decompress(raw, b.unpackSize, b.dictProp)
        out.append((b, plain))
    return out


def test_writer(pkg, codec):
    L = _lib(pkg)
    data = riscv_soup(1_200_000, 71)[:(3 << 20) + 12_345] + call_heavy_riscv(1 << 20, 5)
    c17 = pkg.Codec(0, frame_log=17, window_log=17)
    try:
        for c, F in ((codec, 1 << 20), (c17, 1 << 17)):
            for pc in (0, 0x1000):
                xz = c.xz_compress(data, 4, RISCV, pc)
                r = _ref_unpack(xz, len(data))
                if r:
                    assert r[0] == 0 and r[1] == data and r[3] != 0, (F, pc)
                assert c.xz_decompress(xz) == data, (F, pc)
                blocks = _block_payloads(L, xz)
                assert len(blocks) == (len(data) + F - 1) // F
                for i, (b, filtered) in enumerate(blocks):
                    assert (b.nFilters, b.filterId[0], b.filterProp[0]) == (1, RISCV, pc)
                    assert filtered == oracle_riscv(1, data[i * F:(i + 1) * F], pc), (F, pc, i)
    finally:
        c17.close()
    code = call_heavy_riscv(2 << 20, 3)
    plain = codec.xz_compress(code, 4); bcj = codec.xz_compress(code, 4, RISCV, 0)
    assert len(bcj) < 0.8 * len(plain) and codec.xz_decompress(bcj) == code


def test_reader_on_foreign_files(pkg, codec, soup):
    data = soup[:3_000_001]
    for pc in (0, 0x1000):
        xz = foreign_xz(data, pc)
        r = _ref_unpack(xz, len(data))
        assert r is None or (r[0] == 0 and r[1] == data and r[3] != 0)
        assert codec.xz_decompress(xz) == data, hex(pc)
    two = foreign_xz(data[:100_001], 0) + foreign_xz(data[100_001:], 0x1000)      # the second Block starts at an odd offset
    r = _ref_unpack(two, len(data))
    assert r is None or (r[0] == 0 and r[1] == data)
    assert codec.xz_decompress(two) == data
