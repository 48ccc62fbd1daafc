"""GPU probe: method 21 with the price-based parse -- stage times, ratio and a round trip (needs a GPU)."""
import sys, time, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import __graft_entry__ as g
pkg = g.load_package()
mb = int(sys.argv[1]) if len(sys.argv) > 1 else 256
fl = int(sys.argv[2]) if len(sys.argv) > 2 else 20
sl = int(sys.argv[3]) if len(sys.argv) > 3 else 2
data = pkg.corpus.g2(mb << 20)
for parse in (1, 0):
    c = pkg.Codec(0, frame_log=fl, window_log=fl, lzma2_slice_log=sl, lzma2_parse=parse)
    c.lzma2_compress(data[:8 << 20])
    c.reset_stats()
    t0 = time.time(); prop, comp = c.lzma2_compress(data); dt = time.time() - t0
    print(f"parse={parse} fl={fl} sl={sl} {mb} MiB: host-to-host {dt*1e3:.0f} ms, stage C/M {c.stat(1):.0f} ms, stage P {c.stat(10):.0f} ms, stage R {c.stat(2):.0f} ms, "
          f"assemble {c.stat(3):.0f} ms, ratio {data.nbytes/len(comp):.4f}", flush=True)
    if parse:
        out = c.lzma2_decompress(comp, prop)
        print("roundtrip", np.array_equal(np.frombuffer(out, dtype=np.uint8), data), flush=True)
    c.close()
