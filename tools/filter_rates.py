"""Rates of the GPU filters (b200z_filter_device) on 1 GiB held in device memory, and of the reference's single-thread RISC-V converter
on the host for comparison.  Usage: python tools/filter_rates.py OUT_DIR [--gib 1] [--reps 3]

Every GPU call ends in a stream synchronise, so a host clock around it times the whole call (its staging copy included).  Each timed
call starts from a fresh upload of its input; the upload is not timed.  One untimed call of the same size comes first.
Writes OUT_DIR/filter_rates.json and prints it."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

RISCV, X86, ARM64, DELTA = 0x0B, 0x03030103, 0x0A, 0x03


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True, text=True, check=True).stdout
    lines = [l for l in out.strip().splitlines() if l.strip()]
    return {"query": lines[0], "cards": lines[1:]}


def inputs(n, pkg):
    from test_filters import call_heavy_code, instruction_soup
    from test_riscv_filter import ADVERSARIAL, call_heavy_riscv
    tile = lambda b: np.resize(np.frombuffer(b, dtype=np.uint8), n)
    return [("riscv_call_heavy", RISCV, 0, tile(call_heavy_riscv(4 << 20, 3))),
            ("riscv_adversarial", RISCV, 0, tile(ADVERSARIAL * (1 << 20))),
            ("x86_call_heavy", X86, 0, tile(call_heavy_code(1 << 20, 3))),
            ("arm64_soup", ARM64, 0, tile(instruction_soup(ARM64, 1 << 18, 21))),
            ("delta4_ramp", DELTA, 4, tile(pkg.corpus.entropy_class(2, 4 << 20).tobytes()))]


def ref_riscv_rate(data, reps):
    path = os.path.join(ROOT, "oracle", "_ref", "libref_xz.so")
    if not os.path.exists(path):
        return None
    R = ctypes.CDLL(path)
    res = {}
    for name in ("Enc", "Dec"):
        f = getattr(R, f"z7_BranchConv_RISCV_{name}")
        f.restype = ctypes.c_void_p; f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32]
        best = None
        for _ in range(reps):
            buf = data.copy()
            t0 = time.perf_counter(); f(buf.ctypes.data, buf.nbytes, 0); dt = time.perf_counter() - t0
            best = dt if best is None else min(best, dt)
        res[name.lower() + "_GBps"] = round(data.nbytes / best / 1e9, 3)
    res["bytes"] = int(data.nbytes)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import __graft_entry__ as ge
    pkg = ge.load_package()
    n = int(a.gib * (1 << 30))
    result = {"gpu": gpu_info(), "bytes": n, "reps": a.reps, "gpu_rates": {}}
    c = pkg.Codec(0)
    L = c.L
    d = ctypes.c_void_p()
    c._check(L.b200z_dev_alloc(c.h, ctypes.byref(d), n))
    ref_input = None
    try:
        for name, method, prop, data in inputs(n, pkg):
            row = {}
            for enc in (1, 0):
                src = data
                if not enc:                                         # decode what the GPU encoded
                    c._check(L.b200z_dev_upload(c.h, d, data.ctypes.data, n))
                    c._check(L.b200z_filter_device(c.h, method, 1, d, n, prop))
                    src = np.empty(n, dtype=np.uint8)
                    c._check(L.b200z_dev_download(c.h, src.ctypes.data, d, n))
                    if name == "riscv_call_heavy":
                        ref_input = (data, src)
                c._check(L.b200z_dev_upload(c.h, d, src.ctypes.data, n))
                c._check(L.b200z_filter_device(c.h, method, enc, d, n, prop))          # warm-up
                times = []
                for _ in range(a.reps):
                    c._check(L.b200z_dev_upload(c.h, d, src.ctypes.data, n))
                    t0 = time.perf_counter()
                    c._check(L.b200z_filter_device(c.h, method, enc, d, n, prop))
                    times.append(time.perf_counter() - t0)
                row["enc_GBps" if enc else "dec_GBps"] = round(n / min(times) / 1e9, 2)
                row["enc_ms" if enc else "dec_ms"] = [round(t * 1e3, 3) for t in times]
            result["gpu_rates"][name] = row
            print(name, row, flush=True)
    finally:
        L.b200z_dev_free(c.h, d)
        c.close()
    m = min(n, 256 << 20)
    plain, enc = ref_input
    ref = ref_riscv_rate(plain[:m], a.reps)
    if ref is not None:                                              # the GPU's encoding agrees with the reference's on the slice
        from test_riscv_filter import ref_riscv
        ref["gpu_output_matches_prefix"] = ref_riscv(1, plain[:m].tobytes(), 0)[:m - 8] == enc[:m - 8].tobytes()
    result["ref_riscv_single_thread"] = ref if ref is not None else "oracle/_ref not built"
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "filter_rates.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
