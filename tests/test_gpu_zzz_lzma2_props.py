"""GPU: the LZMA2 encoder at other literal / position context bits (B200Z_P_LZMA2_LC/LP/PB) -- bytes of the oracle statement for
both parses, every model placement, both slice schemes and two frame sizes; round trips through the GPU decoder and liblzma; the
.xz writer; parameter errors; the 7-Zip codec module (tests/cpp/coder_props.cpp) and, where it is built, the reference's own
7-Zip host."""
import lzma
import os
import subprocess

import pytest

import helpers as H
from test_oracle_lzma2_props import GRID, chunk_headers, float_table, oracle_lzma2_compress_props, props_byte, text_with_noise

pytestmark = pytest.mark.gpu
OPT = 0x10
E_PARAM = -3
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "7-zip-zstd_b200")


@pytest.fixture(scope="module")
def payload(pkg):
    return text_with_noise(pkg, 1_300_000)


@pytest.mark.parametrize("fl", [20, 23])
@pytest.mark.parametrize("opt", [0, 1])
@pytest.mark.parametrize("lc,lp,pb", GRID)
def test_gpu_bytes_equal_the_oracle(pkg, payload, lc, lp, pb, opt, fl):
    data = payload if fl == 20 else payload + float_table(n=(1 << 20) // 4)       # 1 MiB frames (two) / one 8 MiB frame
    for sl in (0, 2):
        flags = 1 | (sl << 8) | (OPT if opt else 0)
        want = oracle_lzma2_compress_props(data, lc, lp, pb, frameLog=fl, windowLog=fl, flags=flags)
        for model in (1, 2, 3):
            if model == 3 and lc + lp > 3:
                continue
            c = pkg.Codec(0, frame_log=fl, window_log=fl, lzma2_slice_log=sl, lzma2_parse=opt, lzma2_model=model, lzma2_lc=lc, lzma2_lp=lp, lzma2_pb=pb)
            got = c.lzma2_compress(data)
            assert got == want, (sl, model)
            if model == 1:
                prop, lz = got
                assert all(p == props_byte(lc, lp, pb) for _, p in chunk_headers(lz) if p is not None)
                assert c.lzma2_decompress(lz, prop) == data
                assert lzma.decompress(lz, format=lzma.FORMAT_RAW, filters=[{"id": lzma.FILTER_LZMA2, "dict_size": 1 << fl}]) == data
            c.close()


def test_automatic_placement_and_defaults(pkg, payload):
    """model 0 (automatic placement) at lc + lp = 4 with enough chains to leave shared memory; explicit 2/0/2 = the default bytes"""
    data = payload * 8
    want = oracle_lzma2_compress_props(data, 4, 0, 4, frameLog=20, windowLog=20, flags=1 | (2 << 8))
    c = pkg.Codec(0, lzma2_lc=4, lzma2_lp=0, lzma2_pb=4)
    assert c.lzma2_compress(data) == want
    c.close()
    base = pkg.Codec(0).lzma2_compress(payload)
    assert pkg.Codec(0, lzma2_lc=2, lzma2_lp=0, lzma2_pb=2).lzma2_compress(payload) == base == H.oracle_lzma2_compress(payload, frameLog=20, windowLog=20, flags=1 | (2 << 8))


def test_xz_writer_honours_the_context_bits(pkg, payload):
    c = pkg.Codec(0, lzma2_lc=0, lzma2_lp=2, lzma2_pb=2)
    xz = c.xz_compress(payload, 4)
    assert lzma.decompress(xz, format=lzma.FORMAT_XZ) == payload
    assert c.xz_decompress(xz) == payload
    d = pkg.Codec(0).xz_compress(payload, 4)
    assert xz != d                                                      # the Blocks carry lc0 lp2 pb2 chunks, not the default ones


def test_parameter_errors(pkg):
    c = pkg.Codec(0)
    assert (c.get("lzma2_lc"), c.get("lzma2_lp"), c.get("lzma2_pb")) == (2, 0, 2)
    for name, v in (("lzma2_lc", 5), ("lzma2_lp", 5), ("lzma2_pb", 5), ("lzma2_lc", -1)):
        with pytest.raises(pkg.B200zError) as e:
            c.set(name, v)
        assert e.value.code == E_PARAM
    c.set("lzma2_lc", 3); c.set("lzma2_lp", 2); c.set("lzma2_pb", 1)
    assert (c.get("lzma2_lc"), c.get("lzma2_lp"), c.get("lzma2_pb")) == (3, 2, 1)
    data = b"abc" * 50_000
    for call in (lambda: c.lzma2_compress(data), lambda: c.xz_compress(data, 1)):
        with pytest.raises(pkg.B200zError) as e:                        # lc + lp = 5: refused when the compression starts
            call()
        assert e.value.code == E_PARAM and "lc + lp" in str(e.value)
    c.set("lzma2_lp", 1); c.set("lzma2_model", 3)
    with pytest.raises(pkg.B200zError) as e:                            # lc + lp = 4 and the lock-step kernel
        c.lzma2_compress(data)
    assert e.value.code == E_PARAM and "placement 3" in str(e.value)
    c.set("lzma2_model", 0)
    prop, lz = c.lzma2_compress(data)
    assert c.lzma2_decompress(lz, prop) == data and (prop, lz) == oracle_lzma2_compress_props(data, 3, 1, 1, frameLog=20, windowLog=20, flags=1 | (2 << 8))
    c.close()


@pytest.mark.parametrize("lc,lp,pb", [(0, 2, 2), (4, 0, 4), (1, 2, 3)])
def test_codec_module_sets_the_context_bits(pkg, payload, tmp_path, lc, lp, pb):
    src = tmp_path / "in.bin"; src.write_bytes(payload)
    out = subprocess.run([os.path.join(PKG, "build", "coder_props"), os.path.join(PKG, "libb200z_7z.so"), str(src), str(tmp_path / "p"), str(lc), str(lp), str(pb)],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
    assert out.returncode == 0, out.stdout.decode()[-2000:]
    for ext in ("lzma2", "flzma2"):
        lz = (tmp_path / f"p.{ext}").read_bytes()
        assert all(p == props_byte(lc, lp, pb) for _, p in chunk_headers(lz) if p is not None)
        assert lzma.decompress(lz, format=lzma.FORMAT_RAW, filters=[{"id": lzma.FILTER_LZMA2, "dict_size": 1 << 20}]) == payload
        assert H.oracle_lzma2_decompress(lz, len(payload), 16) == (payload, len(lz))


def test_reference_host_archive_with_lc0_lp2(pkg, payload, tmp_path):
    """7z a -m0=lzma2:lc=0:lp=2:pb=2 inside the reference's own 7-Zip host with the module (as tests/test_ref_7z_host.py sets it
    up), verified by the stock 7zz"""
    import shutil
    from test_ref_7z_host import HOST, REF7Z, STOCK
    subprocess.check_call(["bash", os.path.join(ROOT, "oracle", "build_ref_7z.sh")])
    if not (os.path.exists(HOST) and os.path.exists(STOCK)):
        pytest.skip("oracle/_ref/7z not built (no reference sources here)")
    codecs = os.path.join(REF7Z, "host", "Codecs"); os.makedirs(codecs, exist_ok=True)
    shutil.copy(os.path.join(PKG, "libb200z_7z.so"), os.path.join(codecs, "b200z.so"))
    env = dict(os.environ, LD_LIBRARY_PATH=PKG + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))
    path = tmp_path / "payload.bin"; path.write_bytes(payload)
    arc = str(tmp_path / "a.7z")
    for exe, args in ((HOST, ["a", "-m0=lzma2:lc=0:lp=2:pb=2", arc, str(path)]), (STOCK, ["t", arc])):
        p = subprocess.run([exe, *args], cwd=str(tmp_path), env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        out = p.stdout.decode(errors="replace")
        assert p.returncode == 0 and "Everything is Ok" in out, out[-1500:]
