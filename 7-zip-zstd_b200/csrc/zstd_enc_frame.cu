// zstd_enc_frame.cu -- frame assembly for the block-parallel Zstandard encoder (sm_90a).
//
// Stage E leaves every compressed block (3-byte header + body) in a fixed-stride slot.  Here
//   1. one CTA scans the slot sizes (plus per-frame header/trailer bytes) into output offsets;
//   2. one CTA per block copies its slot to the final position; the CTA of a frame's first
//      block also writes the frame header (and the optional 12-byte skippable size hint that
//      mcmilk's multithreading frame format puts in front of every frame,
//      /root/reference/DOC/Methods-Extern.md:91, C/zstdmt/README.md:9-17).
//
// Replaces (reference, /root/reference/C/zstd/): zstd_compress.c:4695 (ZSTD_writeFrameHeader),
// the ordered flush of zstdmt_compress.c:1488 (ZSTDMT_flushProduced).  Oracle statement:
// oracle/zstd_enc_oracle.c (write_frame_header / b2zo_zstd_compress).
#include "b2z_device.cuh"
#include "b2z_kernels.h"

namespace b2z {

__device__ __forceinline__ uint32_t frame_hdr_bytes(const EncGeom& g) { return ((g.flags & 1u) ? 12u : 0u) + 10u; }

__global__ void __launch_bounds__(1024)
zstd_enc_offsets_kernel(uint64_t srcSize, EncGeom g, const uint32_t* __restrict__ slotSize, uint32_t nBlocks,
                        uint64_t* __restrict__ blockOff, uint64_t* __restrict__ outSize, uint64_t* __restrict__ frameOff) {
    __shared__ uint64_t warpSum[32];
    __shared__ uint64_t carry;
    const uint32_t tid = threadIdx.x, lane = tid & 31u, wid = tid >> 5;
    const uint32_t bpf = 1u << (g.frameLog - 17u);
    const uint32_t hdr = frame_hdr_bytes(g), trailer = (g.flags & 2u) ? 4u : 0u;
    const uint32_t lastBlk = nBlocks - 1u;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (uint32_t b0 = 0; b0 < nBlocks; b0 += 1024u) {
        const uint32_t b = b0 + tid;
        uint64_t v = 0; bool first = false;
        if (b < nBlocks) {
            first = (b % bpf) == 0;
            const bool last = ((b % bpf) == bpf - 1u) || b == lastBlk;
            v = (uint64_t)slotSize[b] + (first ? hdr : 0u) + (last ? trailer : 0u);
        }
        uint64_t x = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint64_t y = __shfl_up_sync(B2Z_FULL, x, d); if (lane >= (uint32_t)d) x += y; }
        if (lane == 31) warpSum[wid] = x;
        __syncthreads();
        if (wid == 0) {
            uint64_t s = warpSum[lane], t = s;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const uint64_t y = __shfl_up_sync(B2Z_FULL, t, d); if (lane >= (uint32_t)d) t += y; }
            warpSum[lane] = t - s;                                   // exclusive per-warp base
        }
        __syncthreads();
        const uint64_t excl = carry + warpSum[wid] + (x - v);
        if (b < nBlocks) {
            blockOff[b] = excl + (first ? hdr : 0u);
            if (first && frameOff) frameOff[b / bpf] = excl;
        }
        __syncthreads();
        if (tid == 1023) carry = excl + v;
        __syncthreads();
    }
    if (tid == 0) {
        *outSize = carry;
        if (frameOff) frameOff[(nBlocks + bpf - 1u) / bpf] = carry;
        blockOff[nBlocks] = carry;
    }
    (void)srcSize;
}

// content checksum of every frame (flag bit1): one thread per frame
__global__ void zstd_enc_checksum_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, EncGeom g, uint32_t* __restrict__ cks, uint32_t nFrames) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nFrames) return;
    const uint64_t f0 = (uint64_t)f << g.frameLog;
    const uint64_t fn = enc_frame_bytes(g, srcSize, f);
    cks[f] = (uint32_t)xxh64_device(src + f0, fn);
}

__global__ void __launch_bounds__(256)
zstd_enc_gather_kernel(uint64_t srcSize, EncGeom g, const uint8_t* __restrict__ slots, const uint32_t* __restrict__ slotSize,
                       const uint64_t* __restrict__ blockOff, uint32_t nBlocks, uint8_t* __restrict__ dst, const uint32_t* __restrict__ cks) {
    const uint32_t b = blockIdx.x, tid = threadIdx.x;
    const uint32_t bpf = 1u << (g.frameLog - 17u);
    const uint8_t* s = slots + (size_t)b * B2Z_SLOT;
    uint8_t* d = dst + blockOff[b];
    const uint32_t n = slotSize[b];
    // head bytes up to 16-byte alignment of the destination, then 16-byte stores fed by
    // unaligned-safe 4-byte reads of the (16-byte aligned) slot
    const uint32_t head = (uint32_t)((16u - ((uintptr_t)d & 15u)) & 15u);
    const uint32_t h = head < n ? head : n;
    if (tid < h) d[tid] = s[tid];
    const uint32_t body = (n - h) & ~15u;
    const uint32_t sh = (h & 3u) * 8u;
    const uint32_t* sw = reinterpret_cast<const uint32_t*>(s + (h & ~3u));
    uint4* dq = reinterpret_cast<uint4*>(d + h);
    for (uint32_t i = tid; i < body / 16u; i += 256u) {
        const uint32_t* q = sw + i * 4u;
        const uint32_t a0 = q[0], a1 = q[1], a2 = q[2], a3 = q[3], a4 = sh ? q[4] : 0u;
        uint4 v;
        v.x = __funnelshift_r(a0, a1, sh); v.y = __funnelshift_r(a1, a2, sh);
        v.z = __funnelshift_r(a2, a3, sh); v.w = __funnelshift_r(a3, a4, sh);
        dq[i] = v;
    }
    for (uint32_t i = h + body + tid; i < n; i += 256u) d[i] = s[i];
    // content checksum after the frame's last block
    if ((g.flags & 2u) && tid == 0 && ((b % bpf) == bpf - 1u || b == nBlocks - 1u)) {
        const uint32_t c = cks[b / bpf];
        d[n] = (uint8_t)c; d[n + 1] = (uint8_t)(c >> 8); d[n + 2] = (uint8_t)(c >> 16); d[n + 3] = (uint8_t)(c >> 24);
    }
    // frame header by the first block's CTA
    if ((b % bpf) == 0 && tid == 0) {
        const uint64_t f = b / bpf;
        const uint64_t fn = enc_frame_bytes(g, srcSize, f);
        const uint32_t lastB = (uint32_t)(((f + 1) * bpf < nBlocks) ? (f + 1) * bpf : nBlocks);
        uint8_t* hp = d - 10;
        if (g.flags & 1u) {
            const uint64_t fsize = (blockOff[lastB - 1u] + slotSize[lastB - 1u] + ((g.flags & 2u) ? 4u : 0u)) - (blockOff[b] - 10u);
            uint8_t* kp = hp - 12;
            kp[0] = 0x50; kp[1] = 0x2A; kp[2] = 0x4D; kp[3] = 0x18; kp[4] = 4; kp[5] = 0; kp[6] = 0; kp[7] = 0;
            kp[8] = (uint8_t)fsize; kp[9] = (uint8_t)(fsize >> 8); kp[10] = (uint8_t)(fsize >> 16); kp[11] = (uint8_t)(fsize >> 24);
        }
        uint32_t wl = 10; while ((1ull << wl) < fn && wl < g.windowLog) wl++;
        hp[0] = 0x28; hp[1] = 0xB5; hp[2] = 0x2F; hp[3] = 0xFD;
        hp[4] = (uint8_t)(0x80u | ((g.flags & 2u) ? 4u : 0u));
        hp[5] = (uint8_t)((wl - 10u) << 3);
        hp[6] = (uint8_t)fn; hp[7] = (uint8_t)(fn >> 8); hp[8] = (uint8_t)(fn >> 16); hp[9] = (uint8_t)(fn >> 24);
    }
}

// Batch mode (many independent files, BASELINE configs[4]): files arrive back to back; every frame is copied to a
// 2^frameLog-aligned slot of the staging buffer so that the frame kernels keep their aligned 8-byte loads.
__global__ void __launch_bounds__(256)
zstd_enc_scatter_kernel(const uint8_t* __restrict__ src, const uint64_t* __restrict__ off, const uint32_t* __restrict__ size,
                        uint32_t frameLog, uint8_t* __restrict__ stage) {
    const uint32_t f = blockIdx.x, n = size[f];
    const uint8_t* s = src + off[f];
    uint64_t* d = reinterpret_cast<uint64_t*>(stage + ((size_t)f << frameLog));
    const uint64_t* sa = reinterpret_cast<const uint64_t*>((uintptr_t)s & ~(uintptr_t)7);
    const uint32_t sh = (uint32_t)((uintptr_t)s & 7u) * 8u;
    const uint32_t nWords = (n + 7u) >> 3;
    for (uint32_t i = threadIdx.x; i < nWords; i += 256u) {
        const uint64_t a = sa[i], b = sh ? sa[i + 1] : 0ull;          // the source buffer carries 64 bytes of slack
        d[i] = sh ? ((a >> sh) | (b << (64u - sh))) : a;
    }
}

#ifndef B2Z_CUEMU
void launch_zstd_enc_scatter(const uint8_t* src, const uint64_t* off, const uint32_t* size, uint32_t nFrames, uint32_t frameLog,
                             uint8_t* stage, cudaStream_t st) {
    if (nFrames) zstd_enc_scatter_kernel<<<nFrames, 256, 0, st>>>(src, off, size, frameLog, stage);
}

void launch_zstd_enc_assemble(const uint8_t* src, uint64_t srcSize, const EncGeom& g, const uint8_t* slots, const uint32_t* slotSize,
                              uint32_t nBlocks, uint64_t* blockOff, uint8_t* dst, uint64_t* outSize, uint64_t* frameOff,
                              uint32_t* cks, cudaStream_t st) {
    if (!nBlocks) return;
    if (g.flags & 2u) { const uint32_t nFrames = (uint32_t)((srcSize + (1ull << g.frameLog) - 1) >> g.frameLog);
                        zstd_enc_checksum_kernel<<<(nFrames + 63) / 64, 64, 0, st>>>(src, srcSize, g, cks, nFrames); }
    zstd_enc_offsets_kernel<<<1, 1024, 0, st>>>(srcSize, g, slotSize, nBlocks, blockOff, outSize, frameOff);
    zstd_enc_gather_kernel<<<nBlocks, 256, 0, st>>>(srcSize, g, slots, slotSize, blockOff, nBlocks, dst, cks);
}
#endif

}  // namespace b2z
