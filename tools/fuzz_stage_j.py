"""Longer differential run of stage J in the host emulation (test infrastructure): reference-written and own frames, intact and damaged, through
the jump kernels forced on every frame with segment sizes of 64 KiB / 128 KiB / 1 GiB; the oracle decoder's verdict and bytes are the bar.
usage: python tools/fuzz_stage_j.py <seed> <seconds>"""
import os, sys, ctypes, random, time
_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path[:0] = [_ROOT, os.path.join(_ROOT, "tests")]
import numpy as np
import __graft_entry__ as ge, helpers as H
pkg=ge.load_package(); E=H.cuemu_library()
vp,u64,u32,i64=ctypes.c_void_p,ctypes.c_uint64,ctypes.c_uint32,ctypes.c_int64
E.emu_zstd_decode_jump.restype=i64; E.emu_zstd_decode_jump.argtypes=[vp,u64,vp,u64,u32,vp]
E.emu_set_jump_seglog.restype=None; E.emu_set_jump_seglog.argtypes=[u32]
seed=int(sys.argv[1]); budget=float(sys.argv[2])
rng=random.Random(seed)
parts=[pkg.corpus.g2(150_000).tobytes(), bytes(140_000), pkg.corpus.entropy_class(1,40_000).tobytes(), b"abcdefg"*9000, pkg.corpus.entropy_class(3,90_000).tobytes(), pkg.corpus.entropy_class(2,60_000).tobytes()]
t0=time.time(); n_mut=0; n_ok=0
while time.time()-t0 < budget:
    rng.shuffle(parts); data=b"".join(parts[:rng.randrange(2,6)]); n=len(data)
    kind=rng.randrange(3)
    if kind==0: comp=H.oracle_compress(data, frameLog=rng.choice([17,18,20]), windowLog=20, flags=rng.choice([1,3]))
    elif kind==1: comp=H.ref_compress(data, level=rng.choice([1,3,5,9]), checksum=rng.randrange(2))
    else: comp=H.ref_compress(data, level=rng.choice([1,3]), checksum=rng.randrange(2), windowLog=rng.choice([14,17]))
    for it in range(12):
        c=bytearray(comp); k=rng.randrange(4)
        if it:
            if k==0: c[rng.randrange(len(c))]^=1<<rng.randrange(8)
            elif k==1: c[rng.randrange(len(c))]=rng.randrange(256)
            elif k==2: c=c[:rng.randrange(1,len(c))]
            else:
                a=rng.randrange(len(c)); c[a:a+rng.randrange(1,6)]=bytes(rng.randrange(256) for _ in range(rng.randrange(1,6)))
        cb=np.frombuffer(bytes(c)+bytes(64),dtype=np.uint8); back=np.zeros(n+64,dtype=np.uint8)
        try: want=H.oracle_decompress(bytes(c), n)
        except ValueError: want=None
        E.emu_set_jump_seglog(rng.choice([16,17,30]))
        r=E.emu_zstd_decode_jump(cb.ctypes.data,len(c),back.ctypes.data,n,2,None)
        n_mut+=1
        assert (r>=0)==(want is not None), (seed, kind, it, k, r)
        if want is not None:
            assert back[:r].tobytes()==want, (seed, kind, it, k); n_ok+=1
print(f"seed {seed}: {n_mut} decodes through stage J ({n_ok} accepted), oracle decoder's verdict and bytes every time")
