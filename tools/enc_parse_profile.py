"""Stage G (zstd_enc_dp_kernel, the level-3 parse) on the bench workload: its time, its rates, and where its cycles go.

  python tools/enc_parse_profile.py [--size-mib 4096] [--reps 3] [--lib LIB] [--out FILE]
  python tools/enc_parse_profile.py --build-clocks DIR       # (no GPU needed) DIR/libb200z.so built with -DB2Z_DP_CLOCKS

Compresses --size-mib MiB of G2 text held on the device with compress_device (what bench.py times): one warm-up, --reps timed
calls with the codec's stage counter stat(10) (stage G between two events), and one more call under torch.profiler for the
per-kernel totals.  The card's name, power limit and SM clocks come from nvidia-smi in the same run.

Rates: input GB/s = positions / stage G time; algorithmic DRAM GB/s counts per position the candidate word read twice (DP pass and
walk, 8 B), the choice byte written once and read once and a 4-byte path-literal mask per 32 positions written and read back
(2.25 B), the input byte read about 2.25 times (DP pass, literal pass, sampled histogram, match extensions) and about 2 B of
sequences and literals (the sequence records are staged, read back and written again by the move): 14.5 B.

--lib points the run at another build (B200Z_LIB).  A library built with -DB2Z_DP_CLOCKS also reports the phase split: every warp
adds its clock64() cycles per phase (histogram, DP loads / DP / choice stores, walk loads / walk / record and mask stores, scan,
move of the records, literal-pass loads / literal stores) and the shares of their sum are printed.  The counters cost registers, so that build's own time is not stage G's time.
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
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

BYTES_PER_POSITION = 8 + 2.25 + 2.25 + 2.0
PHASES = ["hist", "dp_load", "dp", "dp_store", "walk_load", "walk", "walk_store", "scan", "move", "lit_load", "lit"]


def card():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as e:                                          # the timing below does not depend on it
        return f"unavailable: {e}"


def build_clocks(out_dir):
    """libb200z.so with -DB2Z_DP_CLOCKS into out_dir (the flags of build.sh)."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    flags = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-Xcompiler", "-fPIC",
             "-I" + os.path.join(PKG, "csrc"), "-I" + os.path.join(ROOT, "include"), "-DB2Z_DP_CLOCKS"]
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
    ap.add_argument("--lib", default=None, help="another build of libb200z.so")
    ap.add_argument("--build-clocks", metavar="DIR", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.build_clocks:
        build_clocks(a.build_clocks)
        return
    if a.lib:
        os.environ["B200Z_LIB"] = os.path.abspath(a.lib)
    import torch
    import __graft_entry__ as ge
    pkg = ge.load_package()
    lib = ctypes.CDLL(pkg.lib_path())
    clocks = getattr(lib, "b200z_dp_clocks", None)
    n = a.size_mib << 20
    host = torch.empty(n, dtype=torch.uint8).pin_memory()
    pkg.corpus.g2_into(host.data_ptr(), n, threads=os.cpu_count() or 8)
    d_in = host.cuda()
    c = pkg.Codec(0, level=3)
    d_comp = torch.empty(c.compress_bound(n), dtype=torch.uint8, device="cuda")
    m = c.compress_device(d_in.data_ptr(), n, d_comp.data_ptr(), d_comp.numel())     # warm-up (scratch allocations)
    torch.cuda.synchronize()
    rec = {"card": card(), "lib": pkg.lib_path(), "size_mib": a.size_mib, "compressed_bytes": m, "reps": []}
    buf = (ctypes.c_ulonglong * (len(PHASES) + 1))()
    if clocks:
        clocks(buf)                                                 # drop the warm-up's counts
    for _ in range(a.reps):
        c.reset_stats(); torch.cuda.synchronize()
        assert c.compress_device(d_in.data_ptr(), n, d_comp.data_ptr(), d_comp.numel()) == m
        torch.cuda.synchronize()
        rec["reps"].append({"match_ms": c.stat(1), "parse_ms": c.stat(10), "entropy_ms": c.stat(2), "assemble_ms": c.stat(3)})
    if clocks:
        assert clocks(buf) == 0
        tot = sum(buf[:len(PHASES)])
        rec["phase_share"] = {p: round(buf[i] / tot, 4) for i, p in enumerate(PHASES)}
        rec["phase_cycles_per_warp"] = {p: buf[i] / max(1, buf[len(PHASES)]) for i, p in enumerate(PHASES)}
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
    parse_ms = sorted(r["parse_ms"] for r in rec["reps"])[len(rec["reps"]) // 2]
    prof_ms = next((v["ms"] for k, v in kernels.items() if "zstd_enc_dp_kernel" in k), None)
    rec["stage_g"] = {"stat_ms_median": parse_ms, "profiler_ms": prof_ms,
                      "input_GBps": n / 1e9 / (parse_ms / 1e3),
                      "dram_GBps_algorithmic": n * BYTES_PER_POSITION / 1e9 / (parse_ms / 1e3), "bytes_per_position": BYTES_PER_POSITION}
    c.close()
    s = json.dumps(rec, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(s)


if __name__ == "__main__":
    main()
