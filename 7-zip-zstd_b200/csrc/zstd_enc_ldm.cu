// zstd_enc_ldm.cu -- stage L of the Zstandard encoder's long mode (sm_90a): matches up to a window of 128 MiB back, in frames of 8 windows.
//
// The long mode (B200Z_P_LONG; the reference's long=N -> ZSTD_c_enableLongDistanceMatching + windowLog N, ZstdEncoder.cpp:128-146,
// 322-331, algorithm zstd_ldm.c:333-470) keeps stage F as it is -- one CTA per REGION of 2^regionLog bytes, tables in shared
// memory, reach of some tens of KiB -- and adds this stage for what lies further back.  Where the reference walks the input once
// with a rolling hash and a bucketed table that always holds the recent past, this stage is two passes that are each parallel
// over every position of the batch (oracle: zstd_enc_oracle.c ldm_frame):
//   pass 1  every SAMPLE (one position in 128, chosen by the content of its 8 bytes) puts position << 4 | tag into the direct-mapped
//           table of its EPOCH (half a window of the frame) with atomicMin: a table ends up holding the FIRST occurrence of every
//           index in its epoch -- a pure function;
//   pass 2  every sample reads its entry in its own epoch's table and in the two before (together: the window), nearest first; a
//           lower position at most a window back whose 64 bytes verify is a far match.  It is walked back to where the
//           agreement starts (not past the segment start, not onto a lower sample: one owner per position, so the writes do not
//           race) and replaces the candidate word there unless stage F's word is as long and itself verifies 64 bytes.
// Stage G prices the word like any other and extends it by direct comparison when it chooses it.
//
// Work per thread and step: one aligned 8-byte word and its successor -> the 8 overlapping 8-byte values that start in it
// (funnel shifts), 8 sample tests (one 64-bit multiply each); the key, the table access and the verification only for the
// 1-in-128 samples.  Traffic: the input twice (coalesced), one 4-byte atomic / load per sample.
#include "b2z_device.cuh"
#include "b2z_kernels.h"

namespace b2z {

#define B2Z_LDM_THREADS 256

__device__ __forceinline__ uint64_t ldm_ld64(const uint64_t* __restrict__ w8, uint32_t p) {      // the 8 bytes at byte p of the frame
    const uint64_t a = w8[p >> 3];
    const uint32_t sh = (p & 7u) * 8u;
    if (sh == 0u) return a;
    return (a >> sh) | (w8[(p >> 3) + 1u] << (64u - sh));
}
__device__ __forceinline__ bool ldm_same64(const uint64_t* __restrict__ w8, uint32_t a, uint32_t b) {   // B2Z_LDM_MINMATCH equal bytes
#pragma unroll 1
    for (uint32_t k = 0; k < B2Z_LDM_MINMATCH; k += 8u) if (ldm_ld64(w8, a + k) != ldm_ld64(w8, b + k)) return false;
    return true;
}

template <int PASS>
__global__ void __launch_bounds__(B2Z_LDM_THREADS)
zstd_enc_ldm_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, EncGeom g, uint32_t* __restrict__ cand, uint32_t* __restrict__ tables) {
    const uint32_t L = g.ldmLog, E = B2Z_LDM_EPOCHLOG(g.windowLog);
    const uint32_t W = 1u << g.windowLog;
    const uint32_t tagMask = (1u << B2Z_LDM_TAGBITS) - 1u;
    const uint64_t* __restrict__ all8 = reinterpret_cast<const uint64_t*>(src);
    const uint64_t nWords = (srcSize + 7u) >> 3;
    for (uint64_t i = (uint64_t)blockIdx.x * B2Z_LDM_THREADS + threadIdx.x; i < nWords; i += (uint64_t)gridDim.x * B2Z_LDM_THREADS) {
        const uint64_t f = (i << 3) >> g.frameLog, f0 = f << g.frameLog;
        const uint32_t n = enc_frame_bytes(g, srcSize, f);
        if (n < B2Z_LDM_MINMATCH) continue;
        const uint32_t p0 = (uint32_t)((i << 3) - f0), lim = n - B2Z_LDM_MINMATCH + 1u;       // p < lim: 64 bytes at p lie inside the frame
        if (p0 >= lim) continue;
        const uint64_t a = all8[i], b = all8[i + 1u];
        uint32_t hits = 0;
#pragma unroll
        for (uint32_t k = 0; k < 8u; k++) {
            const uint64_t v = k ? (a >> (8u * k)) | (b << (64u - 8u * k)) : a;
            if (p0 + k < lim && b2z_ldm_sampled(v)) hits |= 1u << k;
        }
        if (!hits) continue;
        const uint8_t* __restrict__ fb = src + f0;
        const uint64_t* __restrict__ w8 = reinterpret_cast<const uint64_t*>(fb);
        uint32_t* __restrict__ out = cand + f0;
        const uint64_t ep0 = f0 >> E;                                          // frames are whole epochs: the frame's first table
        for (; hits; hits &= hits - 1u) {
            const uint32_t p = p0 + (uint32_t)__ffs((int)hits) - 1u;
            const uint64_t key = b2z_ldm_key(ldm_ld64(w8, p), ldm_ld64(w8, p + 8u), ldm_ld64(w8, p + 16u), ldm_ld64(w8, p + 24u));
            const uint32_t idx = (uint32_t)(key >> (64u - L)), tag = (uint32_t)(key >> (64u - L - B2Z_LDM_TAGBITS)) & tagMask;
            const uint32_t ep = p >> E;
            if (PASS == 0) { atomicMin(&tables[((ep0 + ep) << L) + idx], ((p - (ep << E)) << B2Z_LDM_TAGBITS) | tag); continue; }
            uint32_t d = 0;
            for (uint32_t back = 0; back <= 2u && back <= ep && !d; back++) {
                const uint32_t e = tables[((ep0 + ep - back) << L) + idx];
                if (e == 0xFFFFFFFFu || (e & tagMask) != tag) continue;
                const uint32_t q = ((ep - back) << E) + (e >> B2Z_LDM_TAGBITS);
                if (q >= p || p - q >= W) continue;                            // the first occurrence itself / beyond the window
                if (ldm_same64(w8, q, p)) d = p - q;
            }
            if (!d) continue;
            uint32_t s0 = p; const uint32_t segStart = p & ~(B2Z_SEG - 1u);
            while (s0 > segStart && s0 > d && fb[s0 - 1u] == fb[s0 - 1u - d] && !b2z_ldm_sampled(ldm_ld64(w8, s0 - 1u))) s0--;
            const uint32_t segEnd = ((p | (B2Z_SEG - 1u)) + 1u) < n ? ((p | (B2Z_SEG - 1u)) + 1u) : n;
            const uint32_t maxLen = segEnd - s0 > B2Z_CAP ? B2Z_CAP : segEnd - s0;
            if (maxLen < B2Z_DP_MINLEN) continue;
            const uint32_t c = out[s0];
            if (c && B2Z_CAND_LEN(c) >= maxLen && (maxLen < B2Z_CAP || ldm_same64(w8, s0 - B2Z_CAND_OFF(c), s0))) continue;
            out[s0] = B2Z_CAND(maxLen, d);
        }
    }
}

#ifndef B2Z_CUEMU
size_t zstd_enc_ldm_table_words(const EncGeom& g, uint64_t srcSize) {       // one table per epoch (frames are whole epochs, the last one may be ragged)
    const uint32_t E = B2Z_LDM_EPOCHLOG(g.windowLog);
    return (size_t)((srcSize + (1ull << E) - 1) >> E) << g.ldmLog;
}

cudaError_t launch_zstd_enc_ldm(const uint8_t* src, uint64_t srcSize, const EncGeom& g, uint32_t* cand, uint32_t* tables, uint32_t smCount, cudaStream_t st) {
    if (srcSize == 0 || !g.ldmLog) return cudaSuccess;
    const uint64_t nWords = (srcSize + 7u) >> 3;
    cudaError_t e = cudaMemsetAsync(tables, 0xFF, zstd_enc_ldm_table_words(g, srcSize) * 4u, st);
    if (e != cudaSuccess) return e;
    uint64_t ctas = (nWords + B2Z_LDM_THREADS - 1) / B2Z_LDM_THREADS;
    if (ctas > (uint64_t)smCount * 8u) ctas = (uint64_t)smCount * 8u;
    zstd_enc_ldm_kernel<0><<<(uint32_t)ctas, B2Z_LDM_THREADS, 0, st>>>(src, srcSize, g, cand, tables);
    zstd_enc_ldm_kernel<1><<<(uint32_t)ctas, B2Z_LDM_THREADS, 0, st>>>(src, srcSize, g, cand, tables);
    return cudaGetLastError();
}
#endif

}  // namespace b2z
