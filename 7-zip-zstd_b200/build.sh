#!/bin/bash
# Build libb200z.so (sm_90a only) and the corpus helper in-tree.  Usage: ./build.sh [-v]
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC -Icsrc -I../include"
[ "$1" = "-v" ] && FLAGS="$FLAGS -Xptxas -v"
mkdir -p build
objs=""
for f in csrc/*.cu; do
  o=build/$(basename "${f%.cu}").o
  if [ ! -f "$o" ] || [ "$f" -nt "$o" ] || [ -n "$(find csrc ../include -name '*.h' -newer "$o" -o -name '*.cuh' -newer "$o")" ]; then
    rm -f "$o"
    $NVCC $FLAGS -c "$f" -o "$o" &
    pids="$pids $!"
  fi
  objs="$objs $o"
done
for p in $pids; do wait $p || { echo "build.sh: compilation FAILED" >&2; exit 1; }; done
$NVCC -shared -gencode arch=compute_90a,code=sm_90a -o libb200z.so $objs -lcudart
gcc -O2 -shared -fPIC -pthread -o corpus/libb200z_corpus.so corpus/g2gen.c
# 7-Zip codec module (ICompressCoder classes + CodecExports) and its C++ test driver
g++ -std=c++17 -O2 -fPIC -shared -Wall -Wno-misleading-indentation codec/ZstdCoders.cpp codec/Lzma2Coders.cpp -I../include -L. -lb200z -Wl,-rpath,'$ORIGIN' -o libb200z_7z.so
g++ -std=c++17 -O2 ../tests/cpp/coder_roundtrip.cpp -ldl -o build/coder_roundtrip
g++ -std=c++17 -O2 ../tests/cpp/coder_props.cpp -ldl -o build/coder_props
echo "built $(pwd)/libb200z.so"
