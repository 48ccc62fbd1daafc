"""The RISC-V branch converter (method / xz filter 0x0B) -- csrc/b2z_filter.cu riscv_*_kernel, rule in b2z_filter_ops.h.
CPU: the oracle's sequential statement (tests/riscv_oracle.c) against the reference's own converter (C/Bra.c
z7_BranchConv_RISCV_Enc / _Dec in oracle/_ref/libref_xz.so); decode(encode(x)) == x; the kernel sources through the host emulation
(tests/cuemu/emu_riscv.cpp), across many CTAs and on the run that keeps the four entry walks apart; per-unit encoding; the .xz container fields.
The GPU tests are in tests/test_gpu_zzz_riscv.py."""
import ctypes
import functools
import glob
import hashlib
import os
import random
import subprocess
import tempfile

import numpy as np

import helpers as H

RISCV = 0x0B
OFFSETS = (0, 0x1000, 0x12345678, 0xFFFFF000, 0xFFFFFFFE)
ADVERSARIAL = b"\x97\x00"                                           # AUIPC x1 whose partner check always fails: a step of 6 everywhere


HERE = os.path.dirname(os.path.abspath(__file__))


@functools.lru_cache(maxsize=None)
def _library(kind):
    """tests/riscv_oracle.c ("oracle") or the kernel sources through tests/cuemu/emu_riscv.cpp ("emu") as a shared library in the
    temporary directory, named by a hash of its sources and command: the tree may be read-only, and concurrent test processes each
    move a finished file into place"""
    if kind == "oracle":
        main, deps = os.path.join(HERE, "riscv_oracle.c"), []
        cmd = [os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-shared", "-Wall"]
    else:
        cu, csrc = os.path.join(HERE, "cuemu"), os.path.join(H.ROOT, "7-zip-zstd_b200", "csrc")
        main = os.path.join(cu, "emu_riscv.cpp")
        deps = sorted(glob.glob(os.path.join(cu, "*.h")) + glob.glob(os.path.join(cu, "shim", "*.h")) + glob.glob(os.path.join(csrc, "*")))
        cmd = [os.environ.get("CXX", "g++"), "-std=c++17", "-O2", "-fPIC", "-shared", "-fno-omit-frame-pointer", "-Wall", "-Wno-unused-function",
               "-Wno-unknown-pragmas", "-Wno-unused-variable", "-I" + os.path.join(cu, "shim"), "-I" + cu, "-I" + csrc, "-x", "c++"]
    h = hashlib.sha256(" ".join(cmd).encode())
    for f in [main] + deps:
        with open(f, "rb") as fh:
            h.update(fh.read())
    out = os.path.join(tempfile.gettempdir(), f"b200z_riscv_{kind}_{h.hexdigest()[:20]}.so")
    if not os.path.exists(out):
        tmp = f"{out}.{os.getpid()}"
        subprocess.check_call(cmd + [main, "-o", tmp])
        os.replace(tmp, out)
    return ctypes.CDLL(out)


def oracle_riscv(enc, data, pc):
    """the oracle's statement on a copy of data"""
    f = _library("oracle").b2zo_riscv
    f.restype = None; f.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32]
    buf = np.frombuffer(bytearray(data) + bytearray(1), dtype=np.uint8)
    f(int(enc), buf.ctypes.data, len(data), pc)
    return buf[:len(data)].tobytes()


def ref_riscv(enc, data, pc):
    """the reference's converter on a copy of data, or None where oracle/_ref is absent"""
    path = os.path.join(H.ROOT, "oracle", "_ref", "libref_xz.so")
    if not os.path.exists(path):
        return None
    R = ctypes.CDLL(path)
    f = R.z7_BranchConv_RISCV_Enc if enc else R.z7_BranchConv_RISCV_Dec
    f.restype = ctypes.c_void_p; f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32]
    buf = np.frombuffer(bytearray(data) + bytearray(1), dtype=np.uint8)     # (+1: a valid pointer for empty input)
    f(buf.ctypes.data, len(data), pc)
    return buf[:len(data)].tobytes()


def _i32(op, rd, rs1, imm12, funct3=0):
    return (op | (rd << 7) | (funct3 << 12) | (rs1 << 15) | ((imm12 & 0xFFF) << 20)) & 0xFFFFFFFF


def _jal(rd, off):
    off &= 0x1FFFFF
    return 0x6F | (rd << 7) | (((off >> 12) & 0xFF) << 12) | (((off >> 11) & 1) << 20) | (((off >> 1) & 0x3FF) << 21) | (((off >> 20) & 1) << 31)


def riscv_soup(n_items, seed):
    """instruction-dense bytes that reach every branch of the rule: 16- and 32-bit instructions at both 2-byte phases, JAL with rd x0 /
    x1 / x5 / others, AUIPC with rd x0 / x2 / others followed by a JALR, load or ADDI on the same or another register or by a 16-bit
    instruction, back-to-back AUIPCs, AUIPC x2 in the shape of an encoded pair, immediates at their sign and range edges"""
    rng = random.Random(seed); out = bytearray()
    imm20 = lambda: rng.choice([0, 1, 0x7FFFF, 0x80000, 0xFFFFF, rng.getrandbits(20)])
    imm12 = lambda: rng.choice([0, 1, 0x7FF, 0x800, 0xFFF, rng.getrandbits(12)])
    reg = lambda: rng.choice([0, 1, 2, 5, rng.randrange(32)])
    for _ in range(n_items):
        r = rng.random()
        if r < 0.15:                                                # compressed (low bits != 11): shifts the phase by 2
            out += (rng.getrandbits(16) & ~3 | rng.randrange(3)).to_bytes(2, "little")
        elif r < 0.3:
            out += (rng.getrandbits(32) | 3).to_bytes(4, "little")
        elif r < 0.45:
            off = rng.choice([0, 2, -2, (1 << 20) - 2, -(1 << 20), rng.getrandbits(21) & ~1])
            out += _jal(rng.choice([0, 1, 5, rng.randrange(32)]), off).to_bytes(4, "little")
        elif r < 0.8:
            rd = reg()
            out += ((imm20() << 12) | (rd << 7) | 0x17).to_bytes(4, "little")
            k = rng.random()
            rs1 = rd if k < 0.6 else reg()
            if k < 0.85:
                op, f3 = rng.choice([(0x67, 0), (0x03, rng.randrange(7)), (0x13, 0)])
                out += _i32(op, reg(), rs1, imm12(), f3).to_bytes(4, "little")
            elif k < 0.93:
                out += (rng.getrandbits(16) & ~3).to_bytes(2, "little")
            # else: the next item follows directly (often another AUIPC)
        elif r < 0.9:                                               # AUIPC x2 with bits 13:12 = 11: the shape of an encoded pair
            top = rng.choice([0, 2, 1, 5, 16, 18, rng.randrange(32)])
            w = (top << 27) | (rng.getrandbits(15) << 12) | (3 << 12) | (2 << 7) | 0x17
            out += w.to_bytes(4, "little") + rng.getrandbits(32).to_bytes(4, "little")
        else:
            out += rng.getrandbits(32).to_bytes(4, "little")
    return bytes(out)


def call_heavy_riscv(n, seed):
    """RV64-like code where the filter pays: an `auipc ra, hi` + `jalr ra, lo(ra)` pair to one of 64 targets among ordinary 32-bit and
    compressed instructions -- the pc-relative offsets all differ, the absolute targets repeat"""
    rng = random.Random(seed); targets = [rng.randrange(0, n) & ~1 for _ in range(64)]
    filler = [_i32(0x13, rng.randrange(32), rng.randrange(32), rng.getrandbits(12)) for _ in range(24)] + [0x00A50533, 0xFE113C23, 0x00813083]
    out = bytearray()
    while len(out) < n - 16:
        r = rng.random()
        if r < 0.25:
            rel = (rng.choice(targets) - len(out)) & 0xFFFFFFFF
            hi = ((rel + 0x800) >> 12) & 0xFFFFF; lo = rel & 0xFFF
            out += ((hi << 12) | (1 << 7) | 0x17).to_bytes(4, "little") + _i32(0x67, 1, 1, lo).to_bytes(4, "little")
        elif r < 0.45:
            out += rng.choice([0x4501, 0x852A, 0x60A2, 0x0141, 0x8082]).to_bytes(2, "little")
        else:
            out += rng.choice(filler).to_bytes(4, "little")
    return bytes(out) + bytes(n - len(out))


def _cases():
    arb = random.Random(5)
    yield from ((n, riscv_soup(8, n)[:n]) for n in range(18))
    yield from ((n, riscv_soup(2000, n)[:n]) for n in (4095, 4096, 4097))
    yield 33_333, riscv_soup(9000, 7)[:33_333]
    yield 40_001, bytes(arb.getrandbits(8) for _ in range(40_001))
    yield 20_001, ADVERSARIAL * 10_000 + b"\x13"


def test_oracle_equals_the_reference():
    for n, data in _cases():
        for pc in OFFSETS:
            enc = oracle_riscv(1, data, pc)
            assert oracle_riscv(0, enc, pc) == data, (n, hex(pc))
            r = ref_riscv(1, data, pc)
            if r is None:
                continue
            assert enc == r, (n, hex(pc))
            assert oracle_riscv(0, data, pc) == ref_riscv(0, data, pc), (n, hex(pc))            # decoding arbitrary bytes
            assert oracle_riscv(0, enc, pc) == ref_riscv(0, enc, pc), (n, hex(pc))


def test_soup_reaches_every_branch():
    """the soup is worth testing on: each kind of position the rule distinguishes converts (or is passed over) many times"""
    data = riscv_soup(30_000, 11)
    enc = oracle_riscv(1, data, 0)
    changed = sum(1 for a, b in zip(data, enc) if a != b)
    assert changed > len(data) // 10
    E = _emu()
    # every position the scan converts, through the emulated kernels' own rule, counted by kind
    kinds = {"jal": 0, "pair": 0, "escape": 0}
    i = 0
    while i + 8 <= len(data) & ~1:
        w0 = int.from_bytes(data[i:i + 4], "little"); w1 = int.from_bytes(data[i + 4:i + 8], "little")
        s = E.emu_riscv_scan(w0, w1)
        if s & 1:
            kinds["jal" if (w0 & 0x7F) == 0x6F else ("pair" if (w0 >> 7) & 0x1F != 2 else "escape")] += 1
        i += s & ~1
    assert min(kinds.values()) > 50, kinds


def _emu():
    E = _library("emu")
    E.emu_riscv_filter.restype = None; E.emu_riscv_filter.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32]
    E.emu_riscv_scan.restype = ctypes.c_uint32; E.emu_riscv_scan.argtypes = [ctypes.c_uint32, ctypes.c_uint32]
    return E


def emu_riscv(E, enc, data, prop, unit_log=0):
    buf = np.frombuffer(bytearray(data) + bytearray(8), dtype=np.uint8)
    E.emu_riscv_filter(enc, buf.ctypes.data, len(data), prop, unit_log)
    return buf[:len(data)].tobytes()


def test_emulated_kernels_equal_the_oracle():
    E = _emu()
    soup = riscv_soup(60_000, 21)                                   # ~250 KB: 16 CTAs of 256 chunks
    adv = ADVERSARIAL * 40_000                                      # 80 KB: five CTAs where the walks from different entries never meet
    late = bytearray(adv); late[len(adv) // 2 + 1] = 0x13           # one byte changed in the middle: the walks merge late
    mixed = soup[:50_000] + adv[:33_334] + soup[50_000:90_001]
    for data in (soup + b"\x01", adv, bytes(late), mixed):
        for pc in (0, 0x00ABC000, 0xFFFFFFFE):
            for enc in (1, 0):
                assert emu_riscv(E, enc, data, pc) == oracle_riscv(enc, data, pc), (len(data), hex(pc), enc)
    assert oracle_riscv(1, adv, 0) == adv                   # the reference converts nothing in the run
    for n in list(range(0, 18)) + [63, 64, 65, 71, 72, 16383, 16384, 16385, 16391, 16392]:     # around chunks and CTA spans
        data = soup[:n]
        for enc in (1, 0):
            assert emu_riscv(E, enc, data, 0x1000) == oracle_riscv(enc, data, 0x1000), (n, enc)
    big = (soup * 70)[:1100 * 16384 + 777]                          # more CTAs than the scan kernel has threads
    for enc in (1, 0):
        assert emu_riscv(E, enc, big, 0x1000) == oracle_riscv(enc, big, 0x1000), enc


def test_emulated_per_unit_encoding():
    """unitLog 12 (the xz writer's Blocks): the scan, the addresses and the limit restart in every 4 KiB unit"""
    E = _emu()
    for data in (riscv_soup(12_000, 31)[:9 * 4096 + 1001], (ADVERSARIAL * 20_000)[:5 * 4096 + 7], riscv_soup(3000, 32)[:3 * 4096]):
        for pc in (0, 0x1000, 0xFFFFFFFE):
            want = b"".join(oracle_riscv(1, data[i:i + 4096], pc) for i in range(0, len(data), 4096))
            assert emu_riscv(E, 1, data, pc, 12) == want, (len(data), hex(pc))


def test_riscv_filter_pays_on_call_heavy_code():
    data = call_heavy_riscv(1 << 20, 3)
    filtered = oracle_riscv(1, data, 0)
    assert oracle_riscv(0, filtered, 0) == data
    r = ref_riscv(1, data, 0)
    assert r is None or r == filtered
    plain = len(H.oracle_lzma2_compress(data)[1]); bcj = len(H.oracle_lzma2_compress(filtered)[1])
    assert bcj < 0.8 * plain, (plain, bcj)


def test_xz_container_with_the_riscv_filter(pkg):
    """Blocks that declare filter 0x0B in front of LZMA2: what b200z_xz_wrap writes is decoded and verified by the reference's
    unpacker and parsed back as (0x0B, start offset); an odd start offset is unsupported, as in the reference (XzDec.c)"""
    from test_xz_container import _lib, _parse, _ref_unpack, _wrap
    L = _lib(pkg); fl = 17; F = 1 << fl
    data = riscv_soup(80_000, 41)[:2 * F + 12_345]
    for fprop in (0, 0x1000):
        filtered = b"".join(oracle_riscv(1, data[i:i + F], fprop) for i in range(0, len(data), F))
        prop, lz = H.oracle_lzma2_compress(filtered, frameLog=fl, windowLog=fl, flags=1)
        xz = _wrap(L, lz, prop, 4, data, fl, RISCV, fprop)
        r = _ref_unpack(xz, len(data))
        if r:
            assert r[0] == 0 and r[1] == data and r[3] != 0, hex(fprop)
        rc, blocks, total = _parse(L, xz)
        assert rc == 0 and total == len(data) and len(blocks) == 3
        assert all(b.nFilters == 1 and b.filterId[0] == RISCV and b.filterProp[0] == fprop for b in blocks)
    prop, lz = H.oracle_lzma2_compress(data[:5000])
    odd = _wrap(L, lz, prop, 4, data[:5000], 20, RISCV, 0x1001)
    assert _parse(L, odd)[0] == -6
    r = _ref_unpack(odd, 5000)
    assert r is None or r[0] != 0


def _vli(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80); v >>= 7
    return bytes(out + bytes([v]))


def foreign_xz(data, pc):
    """a one-Block .xz Stream written without this code base: RISC-V by the reference's converter (the oracle's where oracle/_ref is
    absent), raw LZMA2 from liblzma, and Stream Header, Block Header, Index and Footer assembled here (xz-file-format 2-4); CRC64"""
    import lzma
    import zlib
    from test_xz_container import _crc
    filtered = ref_riscv(1, data, pc)
    if filtered is None:
        filtered = oracle_riscv(1, data, pc)
    lz = lzma.compress(filtered, format=lzma.FORMAT_RAW, filters=[{"id": lzma.FILTER_LZMA2, "preset": 6, "dict_size": 1 << 23}])
    head = b"\x00\x04"                                              # Stream Flags: CRC64
    out = bytearray(b"\xfd7zXZ\x00" + head + zlib.crc32(head).to_bytes(4, "little"))
    filt = b"\x0b" + (b"\x04" + pc.to_bytes(4, "little") if pc else b"\x00") + b"\x21\x01" + bytes([22])     # dict 8 MiB = prop 22
    bh = bytearray(b"\x00\xc1" + _vli(len(lz)) + _vli(len(data)) + filt)
    while (len(bh) + 4) % 4:
        bh.append(0)
    bh[0] = (len(bh) + 4) // 4 - 1
    bh += zlib.crc32(bh).to_bytes(4, "little")
    out += bh + lz + bytes(-len(lz) % 4) + _crc(4, data).to_bytes(8, "little")
    index = bytearray(b"\x00" + _vli(1) + _vli(len(bh) + len(lz) + 8) + _vli(len(data)))
    index += bytes(-len(index) % 4)
    index += zlib.crc32(index).to_bytes(4, "little")
    out += index
    tail = (len(index) // 4 - 1).to_bytes(4, "little") + head
    out += zlib.crc32(tail).to_bytes(4, "little") + tail + b"YZ"
    return bytes(out)


def test_foreign_files_are_accepted_by_the_reference_and_parsed(pkg):
    from test_xz_container import _lib, _parse, _ref_unpack
    L = _lib(pkg)
    data = riscv_soup(40_000, 51)[:150_001]
    for pc in (0, 0x1000, 0x7FFFFFFE):
        xz = foreign_xz(data, pc)
        r = _ref_unpack(xz, len(data))
        if r:
            assert r[0] == 0 and r[1] == data and r[2] == len(xz) and r[3] != 0, hex(pc)
        rc, blocks, total = _parse(L, xz)
        assert rc == 0 and total == len(data) and len(blocks) == 1
        assert (blocks[0].nFilters, blocks[0].filterId[0], blocks[0].filterProp[0]) == (1, RISCV, pc)
