"""GPU tests of the batch pipeline behind the host-pointer calls (csrc/b2z_host_pipeline.cu) and of the serial and device-pointer
batch loops beside it: the output does not depend on the path, and a call that fails leaves no copy behind."""
import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu


def test_lzma2_host_batches(pkg):
    """LZMA2 through the host-pointer call in several batches: one after the other on one worker, through the pipeline on two.  Every
    batch but the last drops its end marker; the stream equals the oracle's and decodes to the input."""
    data = pkg.corpus.g2(20 * (1 << 20) + 4321).tobytes()
    want = helpers.oracle_lzma2_compress(data, frameLog=17, windowLog=17)
    for devs in ([0], [0, 0]):
        c = pkg.Codec(devices=devs, frame_log=17, host_batch_log=22)
        try:
            got = c.lzma2_compress(data)
            assert got == want, devs
            assert c.lzma2_decompress(got[1], got[0]) == data, devs
        finally:
            c.close()


def test_decode_error_mid_pipeline_leaves_no_copy_behind(pkg):
    """A checksum flipped in a middle frame fails a pipelined decode with B200Z_E_CHECKSUM (-8).  Once the call has returned, no
    download into the caller's pinned buffer may still be queued: a sentinel written after the call must survive a device-wide
    synchronise.  The same context then decodes the intact stream.  Whether a copy is still queued when a call that does not wait
    for its copies returns depends on timing, so the sentinel check need not fail on every run of such a build."""
    import torch
    data = pkg.corpus.g2(24 << 20).tobytes()
    enc = pkg.Codec(0, flags=3)
    try:
        comp = enc.compress(data)
        head = enc.compress(data[:12 << 20])                 # frames are independent: the first 12 frames of the stream
    finally:
        enc.close()
    assert comp[:len(head)] == head
    bad = bytearray(comp); bad[len(head) - 1] ^= 0x40        # last byte of frame 11's checksum (of 24 frames, 4 per batch)
    src = torch.frombuffer(bad, dtype=torch.uint8).pin_memory()
    dst = torch.empty(len(data), dtype=torch.uint8).pin_memory()
    for devs in ([0], [0, 0, 0]):
        c = pkg.Codec(devices=devs, flags=3, host_batch_log=22)
        try:
            src.copy_(torch.frombuffer(bad, dtype=torch.uint8))
            with pytest.raises(pkg.B200zError) as e:
                c.decompress_into(src.data_ptr(), src.numel(), dst.data_ptr(), dst.numel())
            assert e.value.code == -8, devs
            dst.fill_(0xA5)
            torch.cuda.synchronize()
            assert bool((dst == 0xA5).all()), devs
            src.copy_(torch.frombuffer(bytearray(comp), dtype=torch.uint8))
            assert c.decompress_into(src.data_ptr(), src.numel(), dst.data_ptr(), dst.numel()) == len(data), devs
            assert dst.numpy().tobytes() == data, devs
        finally:
            c.close()


SMALL = (0, 1, 7, 131073, 777_777)                           # empty, and less than one 1 MiB frame


def test_empty_and_sub_frame_inputs(pkg):
    """Empty and sub-frame inputs through both host-pointer compress calls (one worker and two) and both device-pointer calls:
    the oracle's bytes every time."""
    import torch
    g2 = pkg.corpus.g2(max(SMALL)).tobytes()
    for devs in ([0], [0, 0]):
        c = pkg.Codec(devices=devs)
        try:
            for n in SMALL:
                data = g2[:n]
                assert c.compress(data) == helpers.oracle_compress(data), (devs, n)
                assert c.lzma2_compress(data) == helpers.oracle_lzma2_compress(data), (devs, n)
        finally:
            c.close()
    c = pkg.Codec(0)
    try:
        for n in SMALL:
            data = g2[:n]
            d_src = torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy() if n else np.zeros(16, dtype=np.uint8)).cuda()
            cap = c.compress_bound(n)
            d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
            m = c.compress_device(d_src.data_ptr(), n, d_dst.data_ptr(), cap)
            assert d_dst[:m].cpu().numpy().tobytes() == helpers.oracle_compress(data), n
            cap = c.lzma2_compress_bound(n)
            d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
            m, prop = c.lzma2_compress_device(d_src.data_ptr(), n, d_dst.data_ptr(), cap)
            assert (prop, d_dst[:m].cpu().numpy().tobytes()) == helpers.oracle_lzma2_compress(data), n
    finally:
        c.close()
