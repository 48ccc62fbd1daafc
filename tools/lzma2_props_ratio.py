"""Ratio of the LZMA2 encoder at other literal / position context bits (B200Z_P_LZMA2_LC/LP/PB), measured on the CPU through its
sequential statement compiled for each setting (oracle/props/lz2_props.h; the GPU writes the same bytes), next to the reference's stock LZMA2 encoder at
the same lc / lp / pb where oracle/_ref is built.  Inputs: 1 MiB of G2 text and seeded tables of 2^18 little-endian int32 /
float32 values (tests/test_oracle_lzma2_props.py).  Usage: python tools/lzma2_props_ratio.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import __graft_entry__ as G  # noqa: E402
import helpers as H  # noqa: E402
from test_oracle_lzma2_props import float_table, int_table, oracle_lzma2_compress_props  # noqa: E402

SETTINGS = [(2, 0, 2), (0, 2, 2), (3, 0, 2)]


def main():
    pkg = G.load_package()
    inputs = {"G2 text 1 MiB": pkg.corpus.g2(1 << 20).tobytes(), "int32 table 1 MiB": int_table(), "float32 table 1 MiB": float_table()}
    print(f"{'input':20s} {'lc lp pb':9s} {'greedy':>8s} {'price':>8s} {'ref lzma2 -5':>12s}")
    for name, data in inputs.items():
        for q in SETTINGS:
            row = []
            for opt in (0, 0x10):
                row.append(len(data) / len(oracle_lzma2_compress_props(data, *q, frameLog=20, windowLog=20, flags=1 | (2 << 8) | opt)[1]))
            ref = "-"
            if H.ref_lzma_available():
                ref = f"{len(data) / len(H.ref_lzma2_compress(data, level=5, dict_size=1 << 20, lc=q[0], lp=q[1], pb=q[2])[1]):.4f}"
            print(f"{name:20s} {q[0]}  {q[1]}  {q[2]}   {row[0]:8.4f} {row[1]:8.4f} {ref:>12s}")


if __name__ == "__main__":
    main()
