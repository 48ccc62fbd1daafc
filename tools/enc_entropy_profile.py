"""Where the zstd encoder's time goes on the bench workload, and stage E's split into its three kernels.

  python tools/enc_entropy_profile.py [--size-mib 4096] [--reps 3] [--level 3] [--out FILE]

Compresses --size-mib MiB of G2 text held on the device with compress_device (what bench.py times): one warm-up, --reps timed
calls with the codec's stage counters (stat 1 = match, 10 = parse, 2 = entropy: E1 + E2 + E3, 3 = assembly), and one more call
under torch.profiler for the per-kernel totals.  The card's name, power limit and SM clocks come from nvidia-smi in the same
run.  Set B200Z_LIB to profile another build of the library.  Prints one JSON object (and writes it to --out).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def card():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as e:                                          # the timing below does not depend on it
        return f"unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size-mib", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--level", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    pkg = ge.load_package()
    n = a.size_mib << 20
    host = torch.empty(n, dtype=torch.uint8).pin_memory()
    pkg.corpus.g2_into(host.data_ptr(), n, threads=os.cpu_count() or 8)
    d_in = host.cuda()
    c = pkg.Codec(0, level=a.level)
    d_comp = torch.empty(c.compress_bound(n), dtype=torch.uint8, device="cuda")
    m = c.compress_device(d_in.data_ptr(), n, d_comp.data_ptr(), d_comp.numel())     # warm-up (scratch allocations)
    torch.cuda.synchronize()
    rec = {"card": card(), "lib": pkg.lib_path(), "size_mib": a.size_mib, "level": a.level, "compressed_bytes": m, "reps": []}
    for _ in range(a.reps):
        c.reset_stats(); torch.cuda.synchronize()
        assert c.compress_device(d_in.data_ptr(), n, d_comp.data_ptr(), d_comp.numel()) == m
        torch.cuda.synchronize()
        rec["reps"].append({"match_ms": c.stat(1), "parse_ms": c.stat(10), "entropy_ms": c.stat(2), "assemble_ms": c.stat(3)})
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        c.compress_device(d_in.data_ptr(), n, d_comp.data_ptr(), d_comp.numel())
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            kernels[e.key] = {"ms": t / 1e3, "launches": e.count}
    rec["kernels"] = dict(sorted(kernels.items(), key=lambda kv: -kv[1]["ms"]))
    rec["entropy_ms_median"] = sorted(r["entropy_ms"] for r in rec["reps"])[len(rec["reps"]) // 2]
    c.close()
    s = json.dumps(rec, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(s)


if __name__ == "__main__":
    main()
