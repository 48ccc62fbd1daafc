"""Where the zstd decoder's entropy stage (D1) spends its time on the bench workload.

  python tools/dec_entropy_profile.py [--size-mib 4096] [--reps 3] [--lib LIB] [--out FILE]
  python tools/dec_entropy_profile.py --build-clocks DIR       # (no GPU needed) DIR/libb200z.so built with -DB2Z_D1_CLOCKS

Compresses --size-mib MiB of G2 text with the codec's defaults (what bench.py times), then runs decompress_device: one
warm-up, --reps timed calls with the codec's stage counters (stat 4 = D1, stat 5 = D2 + D3 + verify), and one more call under
torch.profiler for the per-kernel totals.  Beside them: the card (nvidia-smi) and the shape of the compressed stream from a
counting pass over its frames on the host (blocks, literal modes, sequences per block, table logs) -- nothing here comes
from timing.  --lib (or B200Z_LIB) profiles another build of the library.

A library built with -DB2Z_D1_CLOCKS also reports the phase split of the two stream kernels: every stream thread adds its
clock64() cycles per phase (table build, refills, table look-ups and arithmetic, output stores), and the shares of each
kernel's sum are printed.  The counters cost registers and instructions, so that build's own times are not D1's times.
Prints one JSON object (and writes it to --out).
"""
import argparse
import ctypes
import glob
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "7-zip-zstd_b200")
PHASES = ["table", "refill", "decode", "store"]            # D1C_* order in csrc/zstd_dec.cu
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


# ---------------------------------------------------------------- counting pass over the frames (RFC 8878)
def _highbit(v):
    return v.bit_length() - 1


def _read_ncount(buf, off, size, max_log):
    """FSE normalized counts at buf[off:off+size] -> (norm list, table log, bytes used)"""
    v = int.from_bytes(bytes(buf[off:off + size]) + b"\0" * 8, "little")
    pos = 0
    log = (v & 15) + 5; pos = 4
    if log > max_log:
        raise ValueError("accuracy log")
    remaining = 1 << log; norm = []
    while remaining > 0:
        nb = _highbit(remaining + 1) + 1
        T = 1 << (nb - 1); mx = 2 * T - 1 - (remaining + 1)
        bits = (v >> pos) & ((1 << nb) - 1)
        if (bits & (T - 1)) < mx:
            count = bits & (T - 1); pos += nb - 1
        else:
            count = bits
            if count >= T:
                count -= mx
            pos += nb
        p = count - 1
        remaining -= 1 if p < 0 else p
        norm.append(p)
        if p == 0:
            while True:
                rep = (v >> pos) & 3; pos += 2
                norm += [0] * rep
                if rep != 3:
                    break
    return norm, log, (pos + 7) >> 3


def _fse_dtable(norm, log):
    size = 1 << log; high = size - 1; sym = [0] * size; nxt = []
    for s, n in enumerate(norm):
        if n == -1:
            sym[high] = s; high -= 1; nxt.append(1)
        else:
            nxt.append(n)
    step = (size >> 1) + (size >> 3) + 3; pos = 0
    for s, n in enumerate(norm):
        for _ in range(max(n, 0)):
            sym[pos] = s; pos = (pos + step) & (size - 1)
            while pos > high:
                pos = (pos + step) & (size - 1)
    tab = []
    for u in range(size):
        s = sym[u]; ns = nxt[s]; nxt[s] += 1
        nb = log - _highbit(ns)
        tab.append((s, nb, (ns << nb) - size))
    return tab


def _huf_bits(buf, off, size):
    """maxBits of the Huffman description at buf[off:]"""
    hb = buf[off]
    if hb >= 128:
        nw = hb - 127
        w = [(buf[off + 1 + i // 2] & 15) if i & 1 else (buf[off + 1 + i // 2] >> 4) for i in range(nw)]
    else:
        norm, log, used = _read_ncount(buf, off + 1, hb, 6)
        tab = _fse_dtable(norm, log)
        bs = bytes(buf[off + 1 + used:off + 1 + hb]); v = int.from_bytes(bs, "little")
        bitpos = len(bs) * 8 - 8 + _highbit(bs[-1])

        def read(n):
            nonlocal bitpos
            bitpos -= n
            return (v >> bitpos) & ((1 << n) - 1) if bitpos >= 0 else (v << -bitpos) & ((1 << n) - 1)
        s1, s2 = read(log), read(log); w = []
        while True:
            w.append(tab[s1][0]); s1 = tab[s1][2] + read(tab[s1][1])
            if bitpos < 0:
                w.append(tab[s2][0]); break
            w.append(tab[s2][0]); s2 = tab[s2][2] + read(tab[s2][1])
            if bitpos < 0:
                w.append(tab[s1][0]); break
    total = sum(1 << (x - 1) for x in w if x)
    return _highbit(total) + 1


def stream_shape(buf):
    import numpy as np
    n = len(buf); ip = 0
    blocks = {"raw": 0, "rle": 0, "compressed": 0}
    lit_modes = {"raw": 0, "rle": 0, "huffman": 0, "treeless": 0}
    lit_streams4 = 0; lit_bytes = 0; huf_lit_bytes = 0
    nseq = []; seq_modes = {"predefined": 0, "rle": 0, "fse": 0, "repeat": 0}
    logs = {"LL": {}, "OF": {}, "ML": {}}; huf_logs = {}; frames = 0
    while ip + 4 <= n:
        magic = int.from_bytes(buf[ip:ip + 4], "little")
        if (magic & 0xFFFFFFF0) == 0x184D2A50:
            ip += 8 + int.from_bytes(buf[ip + 4:ip + 8], "little"); continue
        assert magic == 0xFD2FB528, "not a zstd frame"
        frames += 1
        fhd = buf[ip + 4]; p = ip + 5
        single = (fhd >> 5) & 1; fcs = fhd >> 6; did = fhd & 3
        p += 0 if single else 1
        p += (0, 1, 2, 4)[did]
        p += (single, 2, 4, 8)[fcs]
        while True:
            bh = int.from_bytes(buf[p:p + 3], "little"); p += 3
            last, btype, bsize = bh & 1, (bh >> 1) & 3, bh >> 3
            if btype == 0:
                blocks["raw"] += 1; p += bsize
            elif btype == 1:
                blocks["rle"] += 1; p += 1
            else:
                blocks["compressed"] += 1
                b0 = buf[p]; lt = b0 & 3; sf = (b0 >> 2) & 3
                v = int.from_bytes(buf[p:p + 5], "little")
                if lt <= 1:
                    hdr, regen = ((1, b0 >> 3), (2, (v >> 4) & 0xFFF), (1, b0 >> 3), (3, (v >> 4) & 0xFFFFF))[sf]
                    csize = regen if lt == 0 else 1; streams = 1
                else:
                    if sf <= 1:
                        hdr, regen, csize, streams = 3, (v >> 4) & 0x3FF, (v >> 14) & 0x3FF, 1 if sf == 0 else 4
                    elif sf == 2:
                        hdr, regen, csize, streams = 4, (v >> 4) & 0x3FFF, (v >> 18) & 0x3FFF, 4
                    else:
                        hdr, regen, csize, streams = 5, (v >> 4) & 0x3FFFF, (v >> 22) & 0x3FFFF, 4
                lit_modes[("raw", "rle", "huffman", "treeless")[lt]] += 1
                lit_bytes += regen
                if lt >= 2:
                    huf_lit_bytes += regen; lit_streams4 += streams == 4
                if lt == 2:
                    hb = _huf_bits(buf, p + hdr, csize); huf_logs[hb] = huf_logs.get(hb, 0) + 1
                q = p + hdr + csize
                c0 = buf[q]
                if c0 < 128:
                    ns, q = c0, q + 1
                elif c0 < 255:
                    ns, q = ((c0 - 128) << 8) + buf[q + 1], q + 2
                else:
                    ns, q = buf[q + 1] + (buf[q + 2] << 8) + 0x7F00, q + 3
                nseq.append(ns)
                if ns:
                    modes = buf[q]; q += 1
                    for t, name, ml in ((0, "LL", 9), (1, "OF", 8), (2, "ML", 9)):
                        m = (modes >> (6 - 2 * t)) & 3
                        seq_modes[("predefined", "rle", "fse", "repeat")[m]] += 1
                        if m == 0:
                            lg = (6, 5, 6)[t]
                        elif m == 1:
                            lg = 0; q += 1
                        elif m == 2:
                            _, lg, used = _read_ncount(buf, q, p + bsize - q, ml); q += used
                        else:
                            continue
                        logs[name][lg] = logs[name].get(lg, 0) + 1
                p += bsize
            if last:
                break
        ip = p + (4 if (fhd >> 2) & 1 else 0)
    a = np.array(nseq, dtype=np.int64) if nseq else np.zeros(1, dtype=np.int64)
    srt = lambda d: {str(k): d[k] for k in sorted(d)}
    return {"frames": frames, "blocks": blocks, "literal_modes": lit_modes, "literal_bytes": lit_bytes, "huffman_literal_bytes": huf_lit_bytes,
            "four_stream_literal_blocks": lit_streams4, "huffman_table_log": srt(huf_logs),
            "sequences": int(a.sum()), "sequences_per_block": {"mean": float(a.mean()), "max": int(a.max())},
            "sequence_table_modes": seq_modes, "fse_table_log": {k: srt(v) for k, v in logs.items()}}


# ---------------------------------------------------------------- GPU
def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return f"nvidia-smi unavailable: {e}"


def build_clocks(out_dir):
    """libb200z.so with -DB2Z_D1_CLOCKS into out_dir (the flags of build.sh)."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    flags = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-Xcompiler", "-fPIC",
             "-I" + os.path.join(PKG, "csrc"), "-I" + os.path.join(ROOT, "include"), "-DB2Z_D1_CLOCKS"]
    os.makedirs(out_dir, exist_ok=True)
    procs, objs = [], []
    for f in sorted(glob.glob(os.path.join(PKG, "csrc", "*.cu"))):
        o = os.path.join(out_dir, os.path.basename(f)[:-3] + ".o")
        procs.append(subprocess.Popen([nvcc, *flags, "-c", f, "-o", o]))
        objs.append(o)
    if any(p.wait() for p in procs):
        raise SystemExit("--build-clocks: compilation failed")
    lib = os.path.join(out_dir, "libb200z.so")
    subprocess.check_call([nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", lib, *objs, "-lcudart"])
    print(lib)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size-mib", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--lib", default=None, help="another build of libb200z.so")
    ap.add_argument("--build-clocks", metavar="DIR", default=None)
    ap.add_argument("--no-shape", action="store_true", help="skip the host counting pass")
    a = ap.parse_args()
    if a.build_clocks:
        build_clocks(a.build_clocks)
        return
    if a.lib:
        os.environ["B200Z_LIB"] = os.path.abspath(a.lib)
    import torch
    import __graft_entry__ as ge
    pkg = ge.load_package()
    clocks = getattr(ctypes.CDLL(pkg.lib_path()), "b200z_d1_clocks", None)
    buf = (ctypes.c_ulonglong * (2 * len(PHASES)))()
    n = a.size_mib << 20
    host = torch.empty(n, dtype=torch.uint8).pin_memory()
    pkg.corpus.g2_into(host.data_ptr(), n, threads=os.cpu_count() or 8)
    d_in = host.cuda()
    c = pkg.Codec(0)
    d_comp = torch.empty(c.compress_bound(n), dtype=torch.uint8, device="cuda")
    d_back = torch.empty(n, dtype=torch.uint8, device="cuda")
    m = c.compress_device(d_in.data_ptr(), n, d_comp.data_ptr(), d_comp.numel())
    assert c.decompress_device(d_comp.data_ptr(), m, d_back.data_ptr(), n) == n          # warm-up (scratch allocations)
    torch.cuda.synchronize()
    rec = {"card": card(), "lib": pkg.lib_path(), "size_mib": a.size_mib, "compressed_bytes": m, "reps": []}
    if clocks:
        clocks(buf)                                                 # drop the warm-up's counts
    for _ in range(a.reps):
        c.reset_stats(); torch.cuda.synchronize()
        assert c.decompress_device(d_comp.data_ptr(), m, d_back.data_ptr(), n) == n
        torch.cuda.synchronize()
        rec["reps"].append({"dec_prepass_ms": c.stat(9), "dec_entropy_ms": c.stat(4), "dec_exec_ms": c.stat(5)})
    assert torch.equal(d_back, d_in), "round trip mismatch"
    if clocks:
        assert clocks(buf) == 0
        for k, name in enumerate(["zstd_dec_lit_streams_kernel", "zstd_dec_seq_streams_kernel"]):
            v = buf[k * len(PHASES):(k + 1) * len(PHASES)]; tot = max(1, sum(v))
            rec.setdefault("phase_share", {})[name] = {p: round(v[i] / tot, 4) for i, p in enumerate(PHASES)}
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        c.decompress_device(d_comp.data_ptr(), m, d_back.data_ptr(), n)
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            kernels[e.key] = {"ms": t / 1e3, "launches": e.count}
    rec["kernels"] = dict(sorted(kernels.items(), key=lambda kv: -kv[1]["ms"]))
    rec["dec_entropy_ms_median"] = sorted(r["dec_entropy_ms"] for r in rec["reps"])[len(rec["reps"]) // 2]
    if not a.no_shape:
        rec["shape"] = stream_shape(d_comp[:m].cpu().numpy().tobytes())
    c.close()
    s = json.dumps(rec, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(s)


if __name__ == "__main__":
    main()
