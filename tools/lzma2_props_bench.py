"""Encode speed of the LZMA2 coder at other literal / position context bits (B200Z_P_LZMA2_LC/LP/PB): device-pointer calls
(b200z_lzma2_compress_device, which ends in a stream synchronise) on 1 GiB of G2 text already in HBM, timed with CUDA events,
median of --reps after one warm-up, for both parses.  Needs a GPU; prints one line per setting and a JSON record.
Usage: python tools/lzma2_props_bench.py [--size-mib 1024] [--reps 3] [--frame-log 20]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as G  # noqa: E402

SETTINGS = [(2, 0, 2), (3, 0, 2), (0, 2, 2), (4, 0, 4)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size-mib", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frame-log", type=int, default=20)
    a = ap.parse_args()
    import torch
    pkg = G.load_package()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip()
    n = a.size_mib << 20
    src = torch.from_numpy(pkg.corpus.g2(n)).cuda()
    rec = {"gpu": gpu, "input": f"{a.size_mib} MiB G2 text", "frame_log": a.frame_log, "results": []}
    print(f"# {gpu}; {a.size_mib} MiB G2, frames of 2^{a.frame_log}, median of {a.reps}")
    for parse in (0, 1):
        for lc, lp, pb in SETTINGS:
            c = pkg.Codec(0, frame_log=a.frame_log, window_log=a.frame_log, lzma2_parse=parse, lzma2_lc=lc, lzma2_lp=lp, lzma2_pb=pb)
            cap = c.lzma2_compress_bound(n)
            dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
            times, size = [], 0
            for r in range(a.reps + 1):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize(); e0.record()
                size, _ = c.lzma2_compress_device(src.data_ptr(), n, dst.data_ptr(), cap)
                e1.record(); torch.cuda.synchronize()
                if r:
                    times.append(e0.elapsed_time(e1) / 1e3)
            t = sorted(times)[len(times) // 2]
            row = {"parse": parse, "lc": lc, "lp": lp, "pb": pb, "seconds": t, "GBps": n / t / 1e9, "ratio": n / size}
            rec["results"].append(row)
            print(f"parse {parse}  lc{lc} lp{lp} pb{pb}: {row['GBps']:.3f} GB/s  ratio {row['ratio']:.4f}  (runs {', '.join(f'{x:.3f}' for x in times)} s)", flush=True)
            del dst; c.close()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
