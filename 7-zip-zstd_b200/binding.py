"""ctypes binding of the C ABI in include/b200z.h (libb200z.so, built in-tree by build.sh).

Host-side mirror of the reference's coder usage (CPP/7zip/Compress/ZstdEncoder.cpp:250-461,
ZstdDecoder.cpp:66-173): one `Codec` = one coder instance bound to one GPU; `compress` /
`decompress` take a whole `Code()` input.  There is no CPU fallback: if the shared library or
a CUDA device is missing, construction raises.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))

P_LEVEL, P_FRAMELOG, P_HASHLOG_L, P_HASHLOG_S, P_WINDOWLOG, P_FLAGS, P_BATCH_LOG = 1, 2, 3, 4, 5, 6, 7
S_ENC_MATCH_MS, S_ENC_ENTROPY_MS, S_ENC_ASSEMBLE_MS, S_DEC_ENTROPY_MS, S_DEC_EXEC_MS = 1, 2, 3, 4, 5
S_KERNEL_LAUNCHES, S_H2D_BYTES, S_D2H_BYTES = 6, 7, 8
S_DEC_PREPASS_MS, S_ENC_PARSE_MS = 9, 10
MAXSEQ = 32768

EXPORTS = [
    "b200z_device_count", "b200z_create", "b200z_create_multi", "b200z_device_list", "b200z_destroy", "b200z_set_param", "b200z_get_param",
    "b200z_last_error", "b200z_get_stat", "b200z_reset_stats", "b200z_zstd_compress_bound",
    "b200z_zstd_compress_device", "b200z_zstd_compress_host", "b200z_zstd_frame_info",
    "b200z_zstd_decompress_device", "b200z_zstd_decompress_host", "b200z_zstd_enc_stage_m", "b200z_zstd_enc_stage_f",
    "b200z_zstd_enc_stage_e", "b200z_dev_alloc", "b200z_dev_free", "b200z_dev_upload", "b200z_dev_download",
    "b200z_host_alloc_pinned", "b200z_host_free_pinned",
]


class B200zError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"b200z error {code}: {msg}")
        self.code = code


def lib_path():
    return os.environ.get("B200Z_LIB") or os.path.join(_HERE, "libb200z.so")      # B200Z_LIB: an experimental build (tools/)


_lib = None


def load_library():
    """Load libb200z.so (fails loudly if it has not been built: run 7-zip-zstd_b200/build.sh)."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} is missing -- build it with 7-zip-zstd_b200/build.sh (no CPU fallback exists)")
    L = ctypes.CDLL(path)
    vp, sz, i64 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int64
    L.b200z_create.argtypes = [ctypes.POINTER(vp), ctypes.c_int]
    L.b200z_create_multi.argtypes = [ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_int), ctypes.c_int]
    L.b200z_device_list.argtypes = [vp, ctypes.POINTER(ctypes.c_int), ctypes.c_int]
    L.b200z_destroy.argtypes = [vp]; L.b200z_destroy.restype = None
    L.b200z_set_param.argtypes = [vp, ctypes.c_int, i64]
    L.b200z_get_param.argtypes = [vp, ctypes.c_int, ctypes.POINTER(i64)]
    L.b200z_last_error.argtypes = [vp]; L.b200z_last_error.restype = ctypes.c_char_p
    L.b200z_get_stat.argtypes = [vp, ctypes.c_int]; L.b200z_get_stat.restype = ctypes.c_double
    L.b200z_reset_stats.argtypes = [vp]; L.b200z_reset_stats.restype = None
    L.b200z_zstd_compress_bound.argtypes = [vp, sz]; L.b200z_zstd_compress_bound.restype = sz
    for name in ("b200z_zstd_compress_device", "b200z_zstd_compress_host", "b200z_zstd_decompress_device", "b200z_zstd_decompress_host"):
        getattr(L, name).argtypes = [vp, vp, sz, vp, sz, ctypes.POINTER(sz)]
    L.b200z_zstd_frame_info.argtypes = [vp, sz, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint32)]
    L.b200z_zstd_enc_stage_m.argtypes = [vp, vp, sz, vp, vp, vp, vp]
    L.b200z_zstd_enc_stage_f.argtypes = [vp, vp, sz, vp]
    L.b200z_zstd_enc_stage_e.argtypes = [vp, vp, sz, vp, vp, vp, vp, vp, sz, vp]
    L.b200z_zstd_compress_batch_bound.argtypes = [vp, sz, ctypes.c_uint32]; L.b200z_zstd_compress_batch_bound.restype = sz
    L.b200z_zstd_compress_batch_host.argtypes = [vp, vp, vp, ctypes.c_uint32, vp, sz, vp]
    L.b200z_zstd_compress_batch_crc_host.argtypes = [vp, vp, vp, ctypes.c_uint32, vp, sz, vp, vp]
    L.b200z_7z_archive_bound.argtypes = [vp, sz, ctypes.c_uint32, sz]; L.b200z_7z_archive_bound.restype = sz
    L.b200z_7z_build_archive.argtypes = [vp, vp, vp, vp, vp, vp, ctypes.c_uint32, ctypes.c_uint32, vp, sz, ctypes.POINTER(sz)]
    L.b200z_7z_write_archive_host.argtypes = [vp, vp, vp, vp, vp, ctypes.c_uint32, vp, sz, ctypes.POINTER(sz)]
    L.b200z_lzma2_compress_bound.argtypes = [vp, sz]; L.b200z_lzma2_compress_bound.restype = sz
    for name in ("b200z_lzma2_compress_device", "b200z_lzma2_compress_host"):
        getattr(L, name).argtypes = [vp, vp, sz, vp, sz, ctypes.POINTER(sz), ctypes.POINTER(ctypes.c_uint32)]
    L.b200z_lzma2_stream_info.argtypes = [vp, sz, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(sz)]
    for name in ("b200z_lzma2_decompress_device", "b200z_lzma2_decompress_host"):
        getattr(L, name).argtypes = [vp, vp, sz, ctypes.c_uint32, vp, sz, ctypes.POINTER(sz)]
    L.b200z_lzma2_enc_stage_cp.argtypes = [vp, vp, sz, vp, vp, vp]
    L.b200z_xz_compress_bound.argtypes = [vp, sz]; L.b200z_xz_compress_bound.restype = sz
    L.b200z_xz_compress_host.argtypes = [vp, vp, sz, vp, sz, ctypes.POINTER(sz), ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32]
    L.b200z_xz_decompress_host.argtypes = [vp, vp, sz, vp, sz, ctypes.POINTER(sz)]
    L.b200z_xz_parse.argtypes = [vp, sz, vp, ctypes.c_uint32, ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint64)]
    for name in ("b200z_crc32_host", "b200z_crc32_device"):
        getattr(L, name).argtypes = [vp, vp, sz, ctypes.POINTER(ctypes.c_uint32)]
    for name in ("b200z_crc64_host", "b200z_crc64_device"):
        getattr(L, name).argtypes = [vp, vp, sz, ctypes.POINTER(ctypes.c_uint64)]
    for name in ("b200z_filter_host", "b200z_filter_device"):
        getattr(L, name).argtypes = [vp, ctypes.c_uint32, ctypes.c_int, vp, sz, ctypes.c_uint32]
    L.b200z_dev_alloc.argtypes = [vp, ctypes.POINTER(vp), sz]
    L.b200z_dev_free.argtypes = [vp, vp]
    L.b200z_dev_upload.argtypes = [vp, vp, vp, sz]
    L.b200z_dev_download.argtypes = [vp, vp, vp, sz]
    L.b200z_host_alloc_pinned.argtypes = [ctypes.POINTER(vp), sz]
    L.b200z_host_free_pinned.argtypes = [vp]
    _lib = L
    return L


def _addr(buf):
    """address + length of a bytes / bytearray / numpy array / torch tensor (host)"""
    if hasattr(buf, "data_ptr"):
        return buf.data_ptr(), buf.numel() * buf.element_size()
    if hasattr(buf, "ctypes"):
        return buf.ctypes.data, buf.nbytes
    if isinstance(buf, (bytes, bytearray)):
        c = (ctypes.c_char * len(buf)).from_buffer_copy(buf) if isinstance(buf, bytes) else (ctypes.c_char * len(buf)).from_buffer(buf)
        return ctypes.addressof(c), len(buf), c
    raise TypeError(type(buf))


class Codec:
    """One coder instance on one GPU (NCompress::NZSTD::CEncoder/CDecoder's engine)."""

    def __init__(self, device=0, devices=None, **params):
        """device: one GPU; devices=[...]: one context over several GPUs (the *_host calls deal batches of frames over them)"""
        self.L = load_library()
        h = ctypes.c_void_p()
        if devices is not None:
            arr = (ctypes.c_int * len(devices))(*devices)
            rc = self.L.b200z_create_multi(ctypes.byref(h), arr, len(devices))
        else:
            rc = self.L.b200z_create(ctypes.byref(h), device)
        if rc:
            raise B200zError(rc, "b200z_create failed (no CUDA device? there is no CPU fallback)")
        self.h = h
        for k, v in params.items():
            self.set(k, v)

    def close(self):
        if getattr(self, "h", None):
            self.L.b200z_destroy(self.h)
            self.h = None

    __del__ = close

    def _check(self, rc):
        if rc:
            raise B200zError(rc, self.L.b200z_last_error(self.h).decode())

    _PARAMS = dict(level=P_LEVEL, frame_log=P_FRAMELOG, hash_log_l=P_HASHLOG_L, hash_log_s=P_HASHLOG_S,
                   window_log=P_WINDOWLOG, flags=P_FLAGS, batch_log=P_BATCH_LOG, host_batch_log=8, chunk_log=9, lzma2_model=10, lzma2_slice_log=11, lzma2_parse=12, zstd_parse=13, long=14, region_log=15, dec_jump=16, dec_jump_seg_log=17)
    # the LZMA2 encoder's literal / position context bits (B200Z_P_LZMA2_LC/LP/PB), kept beside _PARAMS, whose names tests pin
    _LZMA2_CONTEXT_PARAMS = dict(lzma2_lc=18, lzma2_lp=19, lzma2_pb=20)

    def _param_id(self, name):
        return self._PARAMS[name] if name in self._PARAMS else self._LZMA2_CONTEXT_PARAMS[name]

    def set(self, name, value):
        self._check(self.L.b200z_set_param(self.h, self._param_id(name), int(value)))

    def get(self, name):
        v = ctypes.c_int64()
        self._check(self.L.b200z_get_param(self.h, self._param_id(name), ctypes.byref(v)))
        return v.value

    def stat(self, s):
        return self.L.b200z_get_stat(self.h, s)

    def reset_stats(self):
        self.L.b200z_reset_stats(self.h)

    def compress_bound(self, n):
        return self.L.b200z_zstd_compress_bound(self.h, n)

    # ---- host-pointer API (what the 7-Zip coder wrapper calls)
    def compress(self, data) -> bytes:
        import numpy as np
        src = np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) else data
        n = src.nbytes
        out = np.empty(self.compress_bound(n), dtype=np.uint8)
        sz = ctypes.c_size_t()
        self._check(self.L.b200z_zstd_compress_host(self.h, src.ctypes.data if n else None, n, out.ctypes.data, out.nbytes, ctypes.byref(sz)))
        return out[:sz.value].tobytes()

    def compress_batch(self, files):
        """files: list of bytes -> list of compressed bytes (one independent run of frames per file), one GPU call"""
        import numpy as np
        sizes = np.array([len(f) for f in files], dtype=np.uint64)
        src = np.frombuffer(b"".join(files), dtype=np.uint8) if int(sizes.sum()) else np.zeros(1, dtype=np.uint8)
        cap = self.L.b200z_zstd_compress_batch_bound(self.h, int(sizes.sum()), len(files))
        out = np.empty(cap, dtype=np.uint8); offs = np.zeros(len(files) + 1, dtype=np.uint64)
        self._check(self.L.b200z_zstd_compress_batch_host(self.h, src.ctypes.data, sizes.ctypes.data, len(files), out.ctypes.data, cap, offs.ctypes.data))
        return [out[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(files))], out[:int(offs[-1])].tobytes()

    def write_7z(self, files, names, mtimes=None) -> bytes:
        """a complete non-solid .7z archive (method ZSTD, one folder per file) of `files` (list of bytes), one GPU pass"""
        import numpy as np
        sizes = np.array([len(f) for f in files], dtype=np.uint64)
        total = int(sizes.sum())
        src = np.frombuffer(b"".join(files), dtype=np.uint8) if total else np.zeros(1, dtype=np.uint8)
        enc = [n.encode("utf-8") for n in names]
        arr = (ctypes.c_char_p * len(enc))(*enc)
        mt = np.array(mtimes, dtype=np.uint64) if mtimes is not None else None
        cap = self.L.b200z_7z_archive_bound(self.h, total, len(files), sum(len(e) + 1 for e in enc))
        out = np.empty(cap, dtype=np.uint8); n = ctypes.c_size_t()
        self._check(self.L.b200z_7z_write_archive_host(self.h, src.ctypes.data, sizes.ctypes.data, arr, mt.ctypes.data if mt is not None else None, len(files),
                                                       out.ctypes.data, cap, ctypes.byref(n)))
        return out[:n.value].tobytes()

    def compress_into(self, src_ptr, n, dst_ptr, cap):
        sz = ctypes.c_size_t()
        self._check(self.L.b200z_zstd_compress_host(self.h, src_ptr, n, dst_ptr, cap, ctypes.byref(sz)))
        return sz.value

    def decompress(self, data, max_size=None) -> bytes:
        import numpy as np
        src = np.frombuffer(data, dtype=np.uint8)
        if max_size is None:
            cs, nf = ctypes.c_uint64(), ctypes.c_uint32()
            self._check(self.L.b200z_zstd_frame_info(src.ctypes.data, src.nbytes, ctypes.byref(cs), ctypes.byref(nf)))
            max_size = cs.value
        out = np.empty(max(max_size, 1), dtype=np.uint8)
        sz = ctypes.c_size_t()
        self._check(self.L.b200z_zstd_decompress_host(self.h, src.ctypes.data, src.nbytes, out.ctypes.data, max_size, ctypes.byref(sz)))
        return out[:sz.value].tobytes()

    def decompress_into(self, src_ptr, n, dst_ptr, cap):
        sz = ctypes.c_size_t()
        self._check(self.L.b200z_zstd_decompress_host(self.h, src_ptr, n, dst_ptr, cap, ctypes.byref(sz)))
        return sz.value

    # ---- device-pointer API (inputs already resident in HBM; pointers are ints, e.g. tensor.data_ptr())
    def compress_device(self, d_src, n, d_dst, cap):
        sz = ctypes.c_size_t()
        self._check(self.L.b200z_zstd_compress_device(self.h, d_src, n, d_dst, cap, ctypes.byref(sz)))
        return sz.value

    def decompress_device(self, d_src, n, d_dst, cap):
        sz = ctypes.c_size_t()
        self._check(self.L.b200z_zstd_decompress_device(self.h, d_src, n, d_dst, cap, ctypes.byref(sz)))
        return sz.value

    # ---- LZMA2 (method 21): raw chunk stream + the coder's 1-byte dictionary property
    def lzma2_stream_info(self, data):
        """(decoded size, independent blocks, bytes up to and including the end marker) from the chunk headers (host walk)"""
        import numpy as np
        src = np.frombuffer(data, dtype=np.uint8)
        cs, nb, used = ctypes.c_uint64(), ctypes.c_uint32(), ctypes.c_size_t()
        rc = self.L.b200z_lzma2_stream_info(src.ctypes.data if src.nbytes else None, src.nbytes, ctypes.byref(cs), ctypes.byref(nb), ctypes.byref(used))
        if rc:
            raise B200zError(rc, "LZMA2: malformed stream")
        return cs.value, nb.value, used.value

    def lzma2_compress(self, data):
        """-> (dictProp, raw LZMA2 stream)"""
        import numpy as np
        src = np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) else data
        n = src.nbytes
        out = np.empty(self.L.b200z_lzma2_compress_bound(self.h, n), dtype=np.uint8)
        sz, prop = ctypes.c_size_t(), ctypes.c_uint32()
        self._check(self.L.b200z_lzma2_compress_host(self.h, src.ctypes.data if n else None, n, out.ctypes.data, out.nbytes, ctypes.byref(sz), ctypes.byref(prop)))
        return prop.value, out[:sz.value].tobytes()

    def lzma2_compress_into(self, src_ptr, n, dst_ptr, cap):
        sz, prop = ctypes.c_size_t(), ctypes.c_uint32()
        self._check(self.L.b200z_lzma2_compress_host(self.h, src_ptr, n, dst_ptr, cap, ctypes.byref(sz), ctypes.byref(prop)))
        return sz.value, prop.value

    def lzma2_compress_device(self, d_src, n, d_dst, cap):
        sz, prop = ctypes.c_size_t(), ctypes.c_uint32()
        self._check(self.L.b200z_lzma2_compress_device(self.h, d_src, n, d_dst, cap, ctypes.byref(sz), ctypes.byref(prop)))
        return sz.value, prop.value

    def lzma2_compress_bound(self, n):
        return self.L.b200z_lzma2_compress_bound(self.h, n)

    def lzma2_decompress(self, data, dict_prop, max_size=None) -> bytes:
        import numpy as np
        src = np.frombuffer(data, dtype=np.uint8)
        if max_size is None:
            max_size = self.lzma2_stream_info(data)[0]
        out = np.empty(max(max_size, 1), dtype=np.uint8)
        sz = ctypes.c_size_t()
        self._check(self.L.b200z_lzma2_decompress_host(self.h, src.ctypes.data if src.nbytes else None, src.nbytes, dict_prop, out.ctypes.data, max_size, ctypes.byref(sz)))
        return out[:sz.value].tobytes()

    def lzma2_decompress_into(self, src_ptr, n, dict_prop, dst_ptr, cap):
        sz = ctypes.c_size_t()
        self._check(self.L.b200z_lzma2_decompress_host(self.h, src_ptr, n, dict_prop, dst_ptr, cap, ctypes.byref(sz)))
        return sz.value

    def lzma2_decompress_device(self, d_src, n, dict_prop, d_dst, cap):
        sz = ctypes.c_size_t()
        self._check(self.L.b200z_lzma2_decompress_device(self.h, d_src, n, dict_prop, d_dst, cap, ctypes.byref(sz)))
        return sz.value

    # ---- test tap: stage M outputs (same layout as oracle b2zo_zstd_find_sequences)
    def stage_m(self, data):
        import numpy as np
        src = np.frombuffer(data, dtype=np.uint8)
        n = src.nbytes
        nblk = (n + 131071) // 131072
        d = ctypes.c_void_p()
        self._check(self.L.b200z_dev_alloc(self.h, ctypes.byref(d), n + 64))
        try:
            self._check(self.L.b200z_dev_upload(self.h, d, src.ctypes.data, n))
            seqs = np.zeros(nblk * MAXSEQ, dtype=np.uint64)
            nseq = np.zeros(nblk, dtype=np.uint32); nlit = np.zeros(nblk, dtype=np.uint32)
            lits = np.zeros(n, dtype=np.uint8)
            self._check(self.L.b200z_zstd_enc_stage_m(self.h, d, n, seqs.ctypes.data, nseq.ctypes.data, lits.ctypes.data, nlit.ctypes.data))
        finally:
            self.L.b200z_dev_free(self.h, d)
        return seqs, nseq, lits, nlit

    # ---- test tap: stage F candidate words, one per input byte (layout of oracle b2zo_zstd_candidates, frames back to back)
    def stage_f(self, data):
        import numpy as np
        src = np.frombuffer(data, dtype=np.uint8)
        n = src.nbytes
        d = ctypes.c_void_p()
        self._check(self.L.b200z_dev_alloc(self.h, ctypes.byref(d), n + 64))
        try:
            self._check(self.L.b200z_dev_upload(self.h, d, src.ctypes.data, n))
            cand = np.zeros(n, dtype=np.uint32)
            self._check(self.L.b200z_zstd_enc_stage_f(self.h, d, n, cand.ctypes.data))
        finally:
            self.L.b200z_dev_free(self.h, d)
        return cand

    # ---- test tap: stage E alone on given sequences and literals (layout of oracle b2zo_zstd_find_sequences) -> (the coded
    # blocks back to back, their sizes)
    def stage_e(self, src, seqs, nseq, lits, nlit):
        import numpy as np
        src = np.frombuffer(src, dtype=np.uint8) if isinstance(src, (bytes, bytearray, memoryview)) else src
        n = src.nbytes
        nblk = (n + 131071) // 131072
        seqs = np.ascontiguousarray(seqs, dtype=np.uint64); nseq = np.ascontiguousarray(nseq, dtype=np.uint32)
        lits = np.ascontiguousarray(lits, dtype=np.uint8); nlit = np.ascontiguousarray(nlit, dtype=np.uint32)
        if seqs.size < nblk * MAXSEQ or nseq.size < nblk or lits.size < n or nlit.size < nblk:
            raise ValueError("stage_e: arrays smaller than the block layout of the source")
        out = np.empty(n + 3 * nblk, dtype=np.uint8); sizes = np.zeros(nblk, dtype=np.uint32)
        d = ctypes.c_void_p()
        self._check(self.L.b200z_dev_alloc(self.h, ctypes.byref(d), n + 64))
        try:
            self._check(self.L.b200z_dev_upload(self.h, d, src.ctypes.data, n))
            self._check(self.L.b200z_zstd_enc_stage_e(self.h, d, n, seqs.ctypes.data, nseq.ctypes.data, lits.ctypes.data, nlit.ctypes.data,
                                                      out.ctypes.data, out.nbytes, sizes.ctypes.data))
        finally:
            self.L.b200z_dev_free(self.h, d)
        return out[:int(sizes.sum(dtype=np.uint64))].tobytes(), sizes

    # ---- test tap: the price-based LZMA2 parse (lzma2_parse=1): stage C candidate words [n, 4] and stage P sequences
    # (layouts of the oracle's b2zo_lzma2_candidates / b2zo_lzma2_parse_frame, frames back to back)
    def stage_cp(self, data):
        import numpy as np
        src = np.frombuffer(data, dtype=np.uint8)
        n = src.nbytes
        nblk = (n + 131071) // 131072
        d = ctypes.c_void_p()
        self._check(self.L.b200z_dev_alloc(self.h, ctypes.byref(d), n + 64))
        try:
            self._check(self.L.b200z_dev_upload(self.h, d, src.ctypes.data, n))
            cand = np.zeros(max(n, 1) * 4, dtype=np.uint32)
            seqs = np.zeros(nblk * MAXSEQ, dtype=np.uint64); nseq = np.zeros(nblk, dtype=np.uint32)
            self._check(self.L.b200z_lzma2_enc_stage_cp(self.h, d, n, cand.ctypes.data, seqs.ctypes.data, nseq.ctypes.data))
        finally:
            self.L.b200z_dev_free(self.h, d)
        return cand[:n * 4].reshape(-1, 4), seqs, nseq

    # ---- digests and the .xz container (SURVEY.md 8(f) items 4 and 2)
    def crc32(self, data) -> int:
        import numpy as np
        src = np.frombuffer(data, dtype=np.uint8) if len(data) else np.zeros(1, dtype=np.uint8)
        v = ctypes.c_uint32()
        self._check(self.L.b200z_crc32_host(self.h, src.ctypes.data, len(data), ctypes.byref(v)))
        return v.value

    def crc64(self, data) -> int:
        import numpy as np
        src = np.frombuffer(data, dtype=np.uint8) if len(data) else np.zeros(1, dtype=np.uint8)
        v = ctypes.c_uint64()
        self._check(self.L.b200z_crc64_host(self.h, src.ctypes.data, len(data), ctypes.byref(v)))
        return v.value

    def xz_compress(self, data, check=4, filter_id=0, filter_prop=0) -> bytes:
        """-> .xz file bytes: one Block per frame; check 0 none, 1 CRC32, 4 CRC64; filter_id: 0 or a Codec.filter id run in front of LZMA2,
        every Block on its own (filter_prop: delta distance or start offset; RISC-V 0x0B writes xz filter 0x0B)"""
        import numpy as np
        src = np.frombuffer(data, dtype=np.uint8) if len(data) else np.zeros(1, dtype=np.uint8)
        cap = self.L.b200z_xz_compress_bound(self.h, len(data))
        out = np.empty(cap, dtype=np.uint8); sz = ctypes.c_size_t()
        self._check(self.L.b200z_xz_compress_host(self.h, src.ctypes.data if len(data) else None, len(data), out.ctypes.data, cap, ctypes.byref(sz), check, filter_id, filter_prop))
        return out[:sz.value].tobytes()

    def xz_decompress(self, data) -> bytes:
        import numpy as np
        src = np.frombuffer(data, dtype=np.uint8)
        nb, total = ctypes.c_uint32(), ctypes.c_uint64()
        rc = self.L.b200z_xz_parse(src.ctypes.data, src.nbytes, None, 0, ctypes.byref(nb), ctypes.byref(total))
        if rc:
            raise B200zError(rc, "xz: malformed or unsupported container")
        out = np.empty(max(total.value, 1), dtype=np.uint8); sz = ctypes.c_size_t()
        self._check(self.L.b200z_xz_decompress_host(self.h, src.ctypes.data, src.nbytes, out.ctypes.data, total.value, ctypes.byref(sz)))
        return out[:sz.value].tobytes()

    def filter(self, method_id, encode, data, prop=0) -> bytes:
        """Delta (0x03, prop = distance) / branch converters x86 0x03030103, ARM64 0x0A, ARM 0x03030501, ARM Thumb 0x03030701, PPC 0x03030205,
        SPARC 0x03030805, RISC-V 0x0B (prop = start offset; even for RISC-V and Thumb, else B200zError -6).  BCJ2 and IA64: error -6"""
        import numpy as np
        buf = np.frombuffer(bytearray(data), dtype=np.uint8) if len(data) else np.zeros(1, dtype=np.uint8)
        self._check(self.L.b200z_filter_host(self.h, method_id, 1 if encode else 0, buf.ctypes.data, len(data), prop))
        return buf[:len(data)].tobytes()
