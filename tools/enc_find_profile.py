"""Stage F (zstd_enc_find_kernel, the level-3 match finder) on the bench workload: its time, its rate, and where its cycles go.

  python tools/enc_find_profile.py [--size-mib 4096] [--reps 3] [--level 3] [--lib LIB] [--out FILE]
  python tools/enc_find_profile.py --build-clocks DIR       # (no GPU needed) DIR/libb200z.so built with -DB2Z_F_CLOCKS

Compresses --size-mib MiB of G2 text held on the device with compress_device (what bench.py times): one warm-up, --reps timed
calls with the codec's stage counter stat(1) (stage F between two events), and one more call under torch.profiler for the
per-kernel totals.  The card's name, power limit and SM clocks come from nvidia-smi in the same run.

Cycles per turn: a frame of 2^20 positions is 8192 chunks of 128 (one turn each), one CTA per SM walks its frames one after
the other, so a turn lasts stage F's time * SM clock / (turns per SM) -- with the SM clock nvidia-smi reported during the run.

--lib points the run at another build (B200Z_LIB).  A library built with -DB2Z_F_CLOCKS also reports the phase split: every warp
adds its clock64() cycles per phase (wait: for its turn; turn: the table reads and atomics between the barriers; cand: the
compare of the previous iteration's candidates, with whatever is left of their round trip; work: hash, loads, pack, store) and the shares of their sum are printed.  The
counters cost registers and instructions, so that build's own time is not stage F's time.
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

BYTES_PER_POSITION = 1 + 4                                          # the input byte read once, one candidate word written
PHASES = ["wait", "turn", "cand", "work"]
CHUNK = 128                                                         # positions per turn at the default chunkLog 7


def card():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm,count"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as e:                                          # the timing below does not depend on it
        return f"unavailable: {e}"


def build_clocks(out_dir):
    """libb200z.so with -DB2Z_F_CLOCKS into out_dir (the flags of build.sh)."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    flags = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-Xcompiler", "-fPIC",
             "-I" + os.path.join(PKG, "csrc"), "-I" + os.path.join(ROOT, "include"), "-DB2Z_F_CLOCKS"]
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
    clocks = getattr(lib, "b200z_find_clocks", None)
    n = a.size_mib << 20
    host = torch.empty(n, dtype=torch.uint8).pin_memory()
    pkg.corpus.g2_into(host.data_ptr(), n, threads=os.cpu_count() or 8)
    d_in = host.cuda()
    c = pkg.Codec(0, level=a.level)
    d_comp = torch.empty(c.compress_bound(n), dtype=torch.uint8, device="cuda")
    m = c.compress_device(d_in.data_ptr(), n, d_comp.data_ptr(), d_comp.numel())     # warm-up (scratch allocations)
    torch.cuda.synchronize()
    rec = {"card": card(), "level": a.level, "lib": pkg.lib_path(), "size_mib": a.size_mib, "compressed_bytes": m, "reps": []}
    buf = (ctypes.c_ulonglong * (len(PHASES) + 1))()
    if clocks:
        clocks(buf)                                                 # drop the warm-up's counts
    for _ in range(a.reps):
        c.reset_stats(); torch.cuda.synchronize()
        assert c.compress_device(d_in.data_ptr(), n, d_comp.data_ptr(), d_comp.numel()) == m
        torch.cuda.synchronize()
        rec["reps"].append({"match_ms": c.stat(1), "parse_ms": c.stat(10), "entropy_ms": c.stat(2), "assemble_ms": c.stat(3)})
    rec["card_after"] = card()                                      # the SM clock under load, for the cycles per turn
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
    find_ms = sorted(r["match_ms"] for r in rec["reps"])[len(rec["reps"]) // 2]
    prof_ms = next((v["ms"] for k, v in kernels.items() if "zstd_enc_find_kernel" in k), None)
    props = torch.cuda.get_device_properties(0)
    turns_per_sm = n / CHUNK / props.multi_processor_count
    try:
        sm_mhz = float(rec["card_after"].split(",")[3].split()[0])
    except Exception:
        sm_mhz = None
    rec["stage_f"] = {"stat_ms_median": find_ms, "profiler_ms": prof_ms, "sms": props.multi_processor_count,
                      "input_GBps": n / 1e9 / (find_ms / 1e3),
                      "dram_GBps_algorithmic": n * BYTES_PER_POSITION / 1e9 / (find_ms / 1e3), "bytes_per_position": BYTES_PER_POSITION,
                      "ns_per_turn": find_ms * 1e6 / turns_per_sm,
                      "cycles_per_turn": (find_ms * 1e-3 * sm_mhz * 1e6 / turns_per_sm) if sm_mhz else None}
    c.close()
    s = json.dumps(rec, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(s)


if __name__ == "__main__":
    main()
