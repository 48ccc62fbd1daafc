"""CPU: the LZMA2 encoder's literal / position context bits (B200Z_P_LZMA2_LC/LP/PB) in its sequential statement and in the
kernel sources run by the emulator.

  * The statement (oracle/lzma2_enc_oracle.c: stage R; oracle/lzma2_opt_oracle.c: stage P through csrc/b2z_lzma_model.h) is
    written against the compile-time context bits; props_oracle() compiles it once per setting (oracle/props/lz2_props.h).
  * The kernels take the setting at run time: flags bit 15 + bits 16..23 carry the properties byte (b2z_params.h:
    B2Z_FLAG_LZ2_PROPS) to their run-time instantiations, which tests/cuemu/emu_props.cpp runs as sources on the host."""
import atexit
import ctypes
import glob
import lzma
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import helpers as H

OPT = 0x10
GRID = [(0, 0, 0), (3, 0, 2), (4, 0, 4), (0, 4, 0), (1, 2, 3), (0, 2, 2), (2, 0, 2)]


def props_byte(lc, lp, pb):
    return (pb * 5 + lp) * 9 + lc


def props_flags(lc, lp, pb):
    return 0x8000 | (props_byte(lc, lp, pb) << 16)


_built = {}
_build_dir = None


def _workdir():
    global _build_dir
    if _build_dir is None:
        _build_dir = tempfile.mkdtemp(prefix="b2z_lz2props_")
        atexit.register(shutil.rmtree, _build_dir, True)
    return _build_dir


def props_oracle(lc, lp, pb):
    """the oracle (every oracle/*.c, as oracle/Makefile builds liboracle.so) compiled for lc / lp / pb through the forced include
    oracle/props/lz2_props.h, into a temporary directory"""
    key = ("oracle", lc, lp, pb)
    if key not in _built:
        out = os.path.join(_workdir(), f"liboracle_lc{lc}_lp{lp}_pb{pb}.so")
        srcs = sorted(glob.glob(os.path.join(H.ROOT, "oracle", "*.c")))
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-pthread", "-shared", "-Wall", "-Wno-unused-function",
                               "-I" + os.path.join(H.ROOT, "7-zip-zstd_b200", "csrc"), "-include", os.path.join(H.ROOT, "oracle", "props", "lz2_props.h"),
                               f"-DB2ZO_LC={lc}", f"-DB2ZO_LP={lp}", f"-DB2ZO_PB={pb}", "-o", out, *srcs])
        O = ctypes.CDLL(out)
        O.b2zo_lzma2_compress_bound.restype = ctypes.c_size_t
        O.b2zo_lzma2_compress_bound.argtypes = [ctypes.c_size_t, ctypes.POINTER(H.EncParams)]
        O.b2zo_lzma2_compress.restype = ctypes.c_int64
        O.b2zo_lzma2_compress.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(H.EncParams), ctypes.POINTER(ctypes.c_uint32)]
        vp, u32 = ctypes.c_void_p, ctypes.c_uint32
        O.b2zo_lzma2_final_model.restype = ctypes.c_int64
        O.b2zo_lzma2_final_model.argtypes = [vp, u32, ctypes.POINTER(H.EncParams), vp, vp, vp, vp]
        O.b2zo_lzma2_parse_final_model.argtypes = [vp, u32, ctypes.POINTER(H.EncParams), vp, vp, vp, vp]
        _built[key] = O
    return _built[key]


def oracle_lzma2_compress_props(data, lc, lp, pb, **kw):
    """helpers.oracle_lzma2_compress at lc / lp / pb -> (dictProp, raw LZMA2 stream): the bytes the GPU writes with
    B200Z_P_LZMA2_LC/LP/PB set to them (kw: the oracle's parameters; the flags' context-bit field is not read by the oracle)"""
    O = props_oracle(lc, lp, pb); p = H.enc_params(**kw)
    src = np.frombuffer(data, dtype=np.uint8) if len(data) else np.zeros(1, dtype=np.uint8)
    out = np.empty(O.b2zo_lzma2_compress_bound(len(data), ctypes.byref(p)), dtype=np.uint8); prop = ctypes.c_uint32(0)
    r = O.b2zo_lzma2_compress(out.ctypes.data, out.size, src.ctypes.data, len(data), ctypes.byref(p), ctypes.byref(prop))
    assert r > 0, r
    return prop.value, out[:r].tobytes()


def props_emulator():
    """tests/cuemu/emu_props.cpp compiled as tests/cuemu/Makefile compiles emu_kernels.cpp, into a temporary directory"""
    if "emu" not in _built:
        d = os.path.join(H.ROOT, "tests", "cuemu"); out = os.path.join(_workdir(), "libcuemu_props.so")
        subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-fno-omit-frame-pointer", "-Wall",
                               "-Wno-unused-function", "-Wno-unknown-pragmas", "-Wno-unused-variable", "-I" + os.path.join(d, "shim"), "-I" + d,
                               "-I" + os.path.join(H.ROOT, "7-zip-zstd_b200", "csrc"), "-x", "c++", os.path.join(d, "emu_props.cpp"), "-o", out])
        E = ctypes.CDLL(out)
        vp, u32, u64 = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64
        E.emu_props_cand.restype = u64; E.emu_props_cand.argtypes = [vp, u64, u32, u32, u32, vp]
        E.emu_props_parse.restype = u64; E.emu_props_parse.argtypes = [vp, u64, u32, u32, vp, vp, vp]
        E.emu_props_range_and_assemble.restype = ctypes.c_int64
        E.emu_props_range_and_assemble.argtypes = [vp, u64, u32, u32, vp, vp, vp, u64, ctypes.c_int]
        _built["emu"] = E
    return _built["emu"]


def chunk_headers(lz):
    """(control byte, properties byte or None) of every chunk of a raw LZMA2 stream, up to its end marker"""
    out, ip = [], 0
    while lz[ip]:
        c = lz[ip]
        if c <= 2:
            out.append((c, None)); ip += 3 + ((lz[ip + 1] << 8) | lz[ip + 2]) + 1
        else:
            mode = (c >> 5) & 3
            pack = ((lz[ip + 3] << 8) | lz[ip + 4]) + 1
            out.append((c, lz[ip + 5] if mode >= 2 else None)); ip += (6 if mode >= 2 else 5) + pack
    assert ip == len(lz) - 1
    return out


def text_with_noise(pkg, n=700_000):
    """G2 text with incompressible stretches at unaligned positions: raw chunks, and the state resets after them, start at odd
    positions of the frame, where lp > 0 and pb != 2 see the position the decoder keeps (relative to the dictionary reset)"""
    t = pkg.corpus.g2(n).tobytes(); z = pkg.corpus.entropy_class(1, 200_000).tobytes()
    return t[:150_001] + z[:70_003] + t[150_001:400_000] + z[70_003:75_008] + t[400_000:] + z[100_000:166_667] + b"q"


def int_table(seed=7, n=1 << 18):
    """seeded little-endian int32 values of a slowly varying quantity: 32-bit aligned data, the case lc0 lp2 is for"""
    rng = np.random.default_rng(seed)
    return (np.cumsum(rng.integers(-40, 41, n)) + 100_000).astype("<i4").tobytes()


def float_table(seed=11, n=1 << 18):
    rng = np.random.default_rng(seed)
    return (np.cumsum(rng.normal(0, 1, n)) * 0.25 + 10.0).astype("<f4").tobytes()


def check_stream(data, fl, lz, prop, want_props):
    assert H.oracle_lzma2_decompress(lz, len(data), prop) == (data, len(lz))
    filt = [{"id": lzma.FILTER_LZMA2, "dict_size": 1 << fl}]
    assert lzma.decompress(lz, format=lzma.FORMAT_RAW, filters=filt) == data
    if H.ref_lzma_available():
        assert H.ref_lzma2_decompress(lz, len(data), prop) == (data, len(lz))
    hdrs = chunk_headers(lz)
    assert all(p == want_props for c, p in hdrs if p is not None)
    return hdrs


@pytest.mark.parametrize("opt", [False, True])
@pytest.mark.parametrize("sl", [0, 2])
@pytest.mark.parametrize("lc,lp,pb", GRID)
def test_oracle_codes_the_given_context_bits(pkg, lc, lp, pb, sl, opt):
    data = text_with_noise(pkg); fl = 19
    flags = 1 | (sl << 8) | (OPT if opt else 0)
    prop, lz = oracle_lzma2_compress_props(data, lc, lp, pb, frameLog=fl, windowLog=fl, flags=flags)
    hdrs = check_stream(data, fl, lz, prop, props_byte(lc, lp, pb))
    assert any(c in (1, 2) for c, _ in hdrs), "no uncompressed chunk: the noise stretches did not do their job"
    assert any(c >= 0xC0 and c < 0xE0 for c, _ in hdrs) or sl == 0     # state + props resets after raw chunks / at slice starts
    if (lc, lp, pb) == (2, 0, 2):                                      # the defaults compiled in explicitly: the bytes of liboracle.so
        assert (prop, lz) == H.oracle_lzma2_compress(data, frameLog=fl, windowLog=fl, flags=flags)


def test_context_bits_change_the_stream(pkg):
    """the parameters reach the coder: other lc / lp / pb give other (still valid) streams of the same sequences"""
    data = text_with_noise(pkg, 300_000)
    outs = {q: oracle_lzma2_compress_props(data, *q, frameLog=19, windowLog=19, flags=1)[1] for q in GRID}
    assert len(set(outs.values())) == len(GRID)


@pytest.mark.parametrize("lc,lp,pb", [(0, 2, 2), (4, 0, 4), (1, 2, 3), (0, 4, 0)])
def test_simulated_model_equals_the_coders_model_at_other_context_bits(pkg, lc, lp, pb):
    """test_oracle_lzma2_opt.py's claim "stage P prices from the coder's model" at non-default lc / lp / pb: after the same packets
    stage P's model (lzm_commit_*) and stage R's statement hold the same probabilities, state and rep history"""
    O = props_oracle(lc, lp, pb)
    NP = 1848 + (0x300 << (lc + lp))
    for data, fl, sl in ((pkg.corpus.g2(300_000).tobytes() + b"abcd" * 9001, 20, 1), (int_table(n=60_000), 18, 0)):
        n = len(data); src = np.frombuffer(data, dtype=np.uint8)
        p = H.enc_params(frameLog=fl, windowLog=fl, flags=1 | (sl << 8) | OPT)
        nblk = (n + 131071) // 131072
        seqs = np.zeros(nblk * H.MAXSEQ, dtype=np.uint64); nseq = np.zeros(nblk, dtype=np.uint32)
        pP = np.zeros(NP + 8, dtype=np.uint16); cP = np.zeros(5, dtype=np.uint32); pR = np.zeros(NP + 8, dtype=np.uint16); cR = np.zeros(5, dtype=np.uint32)
        O.b2zo_lzma2_parse_final_model(src.ctypes.data, n, ctypes.byref(p), seqs.ctypes.data, nseq.ctypes.data, pP.ctypes.data, cP.ctypes.data)
        resets = O.b2zo_lzma2_final_model(src.ctypes.data, n, ctypes.byref(p), seqs.ctypes.data, nseq.ctypes.data, pR.ctypes.data, cR.ctypes.data)
        slice_bytes = (1 << fl) >> sl
        assert resets == (n + slice_bytes - 1) // slice_bytes
        assert np.array_equal(cP, cR) and np.array_equal(pP, pR)
        assert not pP[NP:].any()                                        # the model is exactly 1848 + (0x300 << (lc + lp)) entries
        assert int((pP[1848:NP] != 1024).sum()) > 200                 # a literal model that has adapted


# ---------------------------------------------------------------- the kernel sources (emulator)
@pytest.fixture(scope="module")
def emu():
    return props_emulator()


@pytest.mark.parametrize("lc,lp,pb,opt", [(0, 2, 2, True), (3, 0, 2, False), (1, 2, 3, True), (4, 0, 4, False), (0, 4, 0, True),
                                          (2, 0, 2, True)])
def test_emulated_kernels_at_other_context_bits(pkg, emu, lc, lp, pb, opt):
    """the run-time instantiations of stage P (lzma2_parse_kernel<true>) and stage R (one chain per warp with the literal model in
    shared and in global memory; the lock-step kernel where lc + lp <= 3) reproduce the oracle's bytes.  (2, 0, 2) with the explicit
    bit runs the run-time instantiations at the defaults: the bytes of the compile-time ones."""
    t = pkg.corpus.g2(200_000).tobytes(); z = pkg.corpus.entropy_class(1, 80_000).tobytes()
    data = t[:90_001] + z[:70_001] + t[90_001:] + b"xy" * 5003; n = len(data); fl = 18; sl = 1
    flags = 1 | (sl << 8) | (OPT if opt else 0) | props_flags(lc, lp, pb)
    src = np.frombuffer(data + bytes(64), dtype=np.uint8)
    F = 1 << fl; nfr = (n + F - 1) // F; bpf = F >> 17
    if opt:
        cand = np.zeros(nfr * F * 4, dtype=np.uint32)
        emu.emu_props_cand(src.ctypes.data, n, fl, flags, 2, cand.ctypes.data)
        seqs = np.zeros(nfr * bpf * H.MAXSEQ, dtype=np.uint64); nseq = np.zeros(nfr * bpf, dtype=np.uint32)
        assert emu.emu_props_parse(src.ctypes.data, n, fl, flags, cand.ctypes.data, seqs.ctypes.data, nseq.ctypes.data) > 0
    else:
        seqs, nseq, _, _ = H.oracle_find_sequences(data, frameLog=fl, windowLog=fl)
    prop, want = oracle_lzma2_compress_props(data, lc, lp, pb, frameLog=fl, windowLog=fl, flags=flags)
    assert any(c in (1, 2) for c, _ in check_stream(data, fl, want, prop, props_byte(lc, lp, pb)))
    if (lc, lp, pb) == (2, 0, 2):
        assert (prop, want) == H.oracle_lzma2_compress(data, frameLog=fl, windowLog=fl, flags=flags & 0x7FFF)
    for glit in (0, 1, 2):
        out = np.zeros(len(want) + 200_000, dtype=np.uint8)
        r = emu.emu_props_range_and_assemble(src.ctypes.data, n, fl, flags, seqs.ctypes.data, nseq.ctypes.data, out.ctypes.data, out.size, glit)
        if glit == 2 and lc + lp > 3:
            assert r == -3                                              # the lock-step kernel's 13-bit queue entries: refused
            continue
        assert r == len(want) and out[:r].tobytes() == want, glit


# ---------------------------------------------------------------- what the context bits do to the ratio (oracle bytes = GPU bytes)
def test_ratio_direction_where_the_margin_is_clear(pkg):
    """lc0 lp2 pb2, the usual setting for 32-bit aligned data, codes a table of little-endian float32 values in clearly fewer bytes
    than the default lc2 lp0 pb2 with either parse, and an int32 table with the greedy parse (the price-based parse codes that one
    as well either way); on text lc3 and lc2 stay within 1 % of each other"""
    fl = 20
    def size(data, flags, q=None):
        return len((oracle_lzma2_compress_props(data, *q, frameLog=fl, windowLog=fl, flags=flags) if q else
                    H.oracle_lzma2_compress(data, frameLog=fl, windowLog=fl, flags=flags))[1])
    for data, flags in ((float_table(), 1), (float_table(), 1 | OPT), (int_table(), 1)):
        d, a = size(data, flags), size(data, flags, (0, 2, 2))
        assert a < 0.97 * d, (flags, a, d)
    text = pkg.corpus.g2(1 << 20).tobytes()
    d, a = size(text, 1), size(text, 1, (3, 0, 2))
    assert abs(a - d) < 0.01 * d


def test_codec_module_refuses_what_the_reference_refuses():
    """kLitContextBits / kLitPosBits / kPosStateBits on LZMA2 and FLZMA2: E_INVALIDARG for lc + lp > 4 (the engine's lc2 counts when
    lc is not given), pb 5, lp 5, lc 9; S_OK for 4/0/4, 0/4/0 and lp2 alone (tests/cpp/coder_props.cpp, no GPU needed)"""
    pkg = os.path.join(H.ROOT, "7-zip-zstd_b200")
    out = subprocess.run([os.path.join(pkg, "build", "coder_props"), os.path.join(pkg, "libb200z_7z.so"), "--props"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=120)
    assert out.returncode == 0 and b"coder props ok" in out.stdout, out.stdout.decode()[-2000:]


def test_binding_context_parameter_ids_match_header(pkg):
    """the binding's lzma2_lc / lzma2_lp / lzma2_pb are the header's B200Z_P_LZMA2_LC/LP/PB, and no other parameter uses those ids"""
    import re
    hdr = open(os.path.join(H.ROOT, "include", "b200z.h")).read()
    ids = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+B200Z_P_([A-Z0-9_]+)\s+(\d+)", hdr)}
    assert pkg.Codec._LZMA2_CONTEXT_PARAMS == dict(lzma2_lc=ids["LZMA2_LC"], lzma2_lp=ids["LZMA2_LP"], lzma2_pb=ids["LZMA2_PB"]) == dict(lzma2_lc=18, lzma2_lp=19, lzma2_pb=20)
    assert not set(pkg.Codec._PARAMS.values()) & set(pkg.Codec._LZMA2_CONTEXT_PARAMS.values())
    assert len(set(ids.values())) == len(ids)
