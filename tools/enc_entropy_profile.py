"""Where the zstd encoder's time goes on the bench workload, and stage E's split into its three kernels.

  python tools/enc_entropy_profile.py [--size-mib 4096] [--reps 3] [--level 3] [--lib LIB] [--out FILE]
  python tools/enc_entropy_profile.py --build-clocks DIR       # (no GPU needed) DIR/libb200z.so built with -DB2Z_E_CLOCKS

Compresses --size-mib MiB of G2 text held on the device with compress_device (what bench.py times): one warm-up, --reps timed
calls with the codec's stage counters (stat 1 = match, 10 = parse, 2 = entropy: E1 + E2 + E3, 3 = assembly), and one more call
under torch.profiler for the per-kernel totals.  The card's name, power limit and SM clocks come from nvidia-smi in the same
run.  --lib (or B200Z_LIB) profiles another build of the library.

A library built with -DB2Z_E_CLOCKS also reports the phase split of E1 and E2: lane 0 of every warp adds its clock64() cycles
per phase, and each kernel's sums (warp-cycles over the timed calls) and their shares are printed.  The counters cost
registers and instructions, so that build's own times are not stage E's times.  Prints one JSON object (and writes it to --out).
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
E1_PHASES = ["lit_hist", "huf_build", "lit_streams", "seq_pass", "tables", "handoff"]     # E1C_* order in csrc/zstd_enc_entropy.cu
E2_PHASES = ["stage", "code_loads", "chain_steps", "word_stores"]                          # E2C_*
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def card():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as e:                                          # the timing below does not depend on it
        return f"unavailable: {e}"


def build_clocks(out_dir):
    """libb200z.so with -DB2Z_E_CLOCKS into out_dir (the flags of build.sh)."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    flags = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-Xcompiler", "-fPIC",
             "-I" + os.path.join(PKG, "csrc"), "-I" + os.path.join(ROOT, "include"), "-DB2Z_E_CLOCKS"]
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
    ap.add_argument("--level", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--lib", default=None, help="another build of libb200z.so")
    ap.add_argument("--build-clocks", metavar="DIR", default=None)
    a = ap.parse_args()
    if a.build_clocks:
        build_clocks(a.build_clocks)
        return
    if a.lib:
        os.environ["B200Z_LIB"] = os.path.abspath(a.lib)
    import torch
    import __graft_entry__ as ge
    pkg = ge.load_package()
    clocks = getattr(ctypes.CDLL(pkg.lib_path()), "b200z_e_clocks", None)
    buf = (ctypes.c_ulonglong * (len(E1_PHASES) + len(E2_PHASES)))()
    n = a.size_mib << 20
    host = torch.empty(n, dtype=torch.uint8).pin_memory()
    pkg.corpus.g2_into(host.data_ptr(), n, threads=os.cpu_count() or 8)
    d_in = host.cuda()
    c = pkg.Codec(0, level=a.level)
    d_comp = torch.empty(c.compress_bound(n), dtype=torch.uint8, device="cuda")
    m = c.compress_device(d_in.data_ptr(), n, d_comp.data_ptr(), d_comp.numel())     # warm-up (scratch allocations)
    torch.cuda.synchronize()
    rec = {"card": card(), "lib": pkg.lib_path(), "size_mib": a.size_mib, "level": a.level, "compressed_bytes": m, "reps": []}
    if clocks:
        clocks(buf)                                                 # drop the warm-up's counts
    for _ in range(a.reps):
        c.reset_stats(); torch.cuda.synchronize()
        assert c.compress_device(d_in.data_ptr(), n, d_comp.data_ptr(), d_comp.numel()) == m
        torch.cuda.synchronize()
        rec["reps"].append({"match_ms": c.stat(1), "parse_ms": c.stat(10), "entropy_ms": c.stat(2), "assemble_ms": c.stat(3)})
    if clocks:
        assert clocks(buf) == 0
        for name, phases, v in (("zstd_enc_tables_kernel", E1_PHASES, buf[:len(E1_PHASES)]),
                                ("zstd_enc_chains_kernel", E2_PHASES, buf[len(E1_PHASES):])):
            tot = max(1, sum(v))
            rec.setdefault("phase_warp_cycles", {})[name] = {p: int(v[i]) // a.reps for i, p in enumerate(phases)}
            rec.setdefault("phase_share", {})[name] = {p: round(v[i] / tot, 4) for i, p in enumerate(phases)}
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
