// b2z_crc.cu -- CRC32 and CRC64 of device buffers (sm_90a): the digests the archive layer computes over every byte next to the
// coders -- 7-Zip's CRC32 of each file / folder (C/7zCrc.c:298 CrcCalc, CPP/7zip/Common/InStreamWithCRC.cpp) and xz's CRC64 block
// check (C/XzCrc64.c, C/Xz.h:34 XZ_CHECK_CRC64).  SURVEY.md 8(f) item 4: once the coder is fast the host's CRC is the bottleneck.
//
//   crc_pieces_kernel  one THREAD per piece (a fixed 64 KiB for whole-buffer digests, or a caller-given range such as an xz
//                      block): slicing-by-8 over the piece with the eight 256-entry tables in shared memory (built by the CTA
//                      from the polynomial).  The reflected polynomials and the init / final-xor convention are the standard
//                      ones: CRC-32 0xEDB88320, CRC-64/XZ 0xC96C5795D7870F42, init = final xor = all ones.
//   host               a whole-buffer digest = the pieces' digests folded with crc(A || B) = crc(A) * x^(8 |B|) + crc(B) over
//                      GF(2)[x] mod P (the linearity zlib's crc32_combine uses; polynomial arithmetic below is ours).
// Oracle statement: oracle/crc_oracle.c (bit-at-a-time), pinned to the check values of both CRCs, zlib and the reference's CrcCalc / Crc64Update.
#include "b2z_device.cuh"
#ifndef B2Z_CUEMU          // the host emulation build (tests/cuemu) compiles the kernel only
#include <vector>
#include "b2z_ctx.h"
#endif

namespace b2z {

#define B2Z_CRC_PIECE_LOG 16u

// piece i = bytes [off[i], off[i] + len[i]) of src when off != null, else the i-th 2^pieceLog bytes of [0, n)
template <typename T>
__global__ void __launch_bounds__(128)
crc_pieces_kernel(const uint8_t* __restrict__ src, uint64_t n, uint32_t pieceLog, const uint64_t* __restrict__ off, const uint64_t* __restrict__ len,
                  uint32_t nPieces, T poly, T* __restrict__ out) {
    __shared__ T tab[8][256];
    for (uint32_t i = threadIdx.x; i < 256u; i += blockDim.x) {
        T r = (T)i;
        for (int k = 0; k < 8; k++) r = (r >> 1) ^ (poly & ((T)0 - (r & 1)));
        tab[0][i] = r;
    }
    __syncthreads();
    for (uint32_t k = 1; k < 8u; k++) {
        for (uint32_t i = threadIdx.x; i < 256u; i += blockDim.x) { const T r = tab[k - 1][i]; tab[k][i] = tab[0][(uint32_t)(r & 0xFF)] ^ (r >> 8); }
        __syncthreads();
    }
    const uint32_t piece = blockIdx.x * blockDim.x + threadIdx.x;
    if (piece >= nPieces) return;
    uint64_t p0, pl;
    if (off) { p0 = off[piece]; pl = len[piece]; }
    else { p0 = (uint64_t)piece << pieceLog; pl = (n - p0) < (1ull << pieceLog) ? (n - p0) : (1ull << pieceLog); }
    const uint8_t* p = src + p0;
    T crc = ~(T)0;
    uint64_t i = 0;
    for (; i < pl && ((uintptr_t)(p + i) & 7u); i++) crc = tab[0][(uint32_t)((crc ^ p[i]) & 0xFF)] ^ (crc >> 8);
    for (; i + 8 <= pl; i += 8) {
        const uint64_t w = __ldg(reinterpret_cast<const uint64_t*>(p + i)) ^ (uint64_t)crc;
        // (a 32-bit crc is consumed entirely by the xor into the low half of the word)
        T r = tab[7][(uint32_t)(w & 0xFF)] ^ tab[6][(uint32_t)((w >> 8) & 0xFF)] ^ tab[5][(uint32_t)((w >> 16) & 0xFF)] ^ tab[4][(uint32_t)((w >> 24) & 0xFF)]
            ^ tab[3][(uint32_t)((w >> 32) & 0xFF)] ^ tab[2][(uint32_t)((w >> 40) & 0xFF)] ^ tab[1][(uint32_t)((w >> 48) & 0xFF)] ^ tab[0][(uint32_t)(w >> 56)];
        crc = r;
    }
    for (; i < pl; i++) crc = tab[0][(uint32_t)((crc ^ p[i]) & 0xFF)] ^ (crc >> 8);
    out[piece] = ~crc;
}

// ---- SHA-256 (FIPS 180-4) of caller-given ranges, one THREAD per range: the third check type of an xz Block (C/Xz.h:35 XZ_CHECK_SHA256,
// C/Sha256.c).  A range is hashed sequentially (the compression function chains), ranges run in parallel; digests leave as 8 big-endian
// words = the 32 bytes in file order.
__device__ __forceinline__ uint32_t sha_rotr(uint32_t x, uint32_t n) { return (x >> n) | (x << (32u - n)); }
__constant__ uint32_t c_sha256_k[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
    0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
    0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85, 0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
    0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2 };
__device__ inline void sha256_block(uint32_t h[8], const uint8_t* blk) {
    uint32_t w[64];
    for (int i = 0; i < 16; i++) w[i] = ((uint32_t)blk[4 * i] << 24) | ((uint32_t)blk[4 * i + 1] << 16) | ((uint32_t)blk[4 * i + 2] << 8) | blk[4 * i + 3];
    for (int i = 16; i < 64; i++) {
        const uint32_t s0 = sha_rotr(w[i - 15], 7) ^ sha_rotr(w[i - 15], 18) ^ (w[i - 15] >> 3), s1 = sha_rotr(w[i - 2], 17) ^ sha_rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
        w[i] = w[i - 16] + s0 + w[i - 7] + s1;
    }
    uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
    for (int i = 0; i < 64; i++) {
        const uint32_t t1 = hh + (sha_rotr(e, 6) ^ sha_rotr(e, 11) ^ sha_rotr(e, 25)) + ((e & f) ^ (~e & g)) + c_sha256_k[i] + w[i];
        const uint32_t t2 = (sha_rotr(a, 2) ^ sha_rotr(a, 13) ^ sha_rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
        hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}
__global__ void __launch_bounds__(64)
sha256_pieces_kernel(const uint8_t* __restrict__ src, const uint64_t* __restrict__ off, const uint64_t* __restrict__ len, uint32_t nPieces, uint32_t* __restrict__ out /* [nPieces][8] */) {
    const uint32_t piece = blockIdx.x * blockDim.x + threadIdx.x;
    if (piece >= nPieces) return;
    const uint8_t* p = src + off[piece]; const uint64_t n = len[piece];
    uint32_t h[8] = { 0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19 };
    uint64_t i = 0;
    for (; i + 64 <= n; i += 64) sha256_block(h, p + i);
    uint8_t tail[128]; uint32_t t = 0;
    for (; i < n; i++) tail[t++] = p[i];
    tail[t++] = 0x80;
    const uint32_t padTo = t <= 56u ? 56u : 120u;
    while (t < padTo) tail[t++] = 0;
    const uint64_t bits = n * 8u;
    for (int k = 7; k >= 0; k--) tail[t++] = (uint8_t)(bits >> (8 * k));
    sha256_block(h, tail);
    if (t == 128u) sha256_block(h, tail + 64);
    for (int k = 0; k < 8; k++) out[(size_t)piece * 8u + k] = h[k];
}

#ifndef B2Z_CUEMU
cudaError_t launch_sha256_pieces(const uint8_t* src, const uint64_t* off, const uint64_t* len, uint32_t nPieces, uint32_t* out, cudaStream_t st) {
    if (!nPieces) return cudaSuccess;
    sha256_pieces_kernel<<<(nPieces + 63u) / 64u, 64, 0, st>>>(src, off, len, nPieces, out);
    return cudaGetLastError();
}

// ---- GF(2) polynomial arithmetic mod P, reflected bit order (bit W-1 = x^0); W = 32 or 64
template <typename T> static T gf_mul(T a, T b, T poly) {
    const T top = (T)1 << (sizeof(T) * 8 - 1);
    T p = 0;
    for (T m = top; m; m >>= 1) {
        if (a & m) p ^= b;
        b = (b & 1) ? (b >> 1) ^ poly : b >> 1;                      // b *= x
    }
    return p;
}
// x^(8 * bytes) mod P
template <typename T> static T gf_xpow8(uint64_t bytes, T poly) {
    const T top = (T)1 << (sizeof(T) * 8 - 1);
    T r = top;                                                      // x^0
    T sq = top >> 1;                                                // x^1
    for (int k = 0; k < 3; k++) sq = gf_mul(sq, sq, poly);          // x^8
    for (; bytes; bytes >>= 1) { if (bytes & 1) r = gf_mul(r, sq, poly); sq = gf_mul(sq, sq, poly); }
    return r;
}
template <typename T> static T crc_fold(const std::vector<T>& pieces, uint64_t n, uint32_t pieceLog, T poly) {
    if (pieces.empty()) return 0;                                   // crc of the empty message: ~(~0) = 0
    const T full = gf_xpow8<T>(1ull << pieceLog, poly);
    T crc = pieces[0];
    for (size_t i = 1; i < pieces.size(); i++) {
        const uint64_t pl = (i + 1 == pieces.size()) ? n - ((uint64_t)i << pieceLog) : (1ull << pieceLog);
        crc = gf_mul(crc, pl == (1ull << pieceLog) ? full : gf_xpow8<T>(pl, poly), poly) ^ pieces[i];
    }
    return crc;
}

template <typename T> cudaError_t launch_crc_pieces(const uint8_t* src, uint64_t n, uint32_t pieceLog, const uint64_t* off, const uint64_t* len,
                                                    uint32_t nPieces, T poly, T* out, cudaStream_t st) {
    if (!nPieces) return cudaSuccess;
    crc_pieces_kernel<T><<<(nPieces + 127u) / 128u, 128, 0, st>>>(src, n, pieceLog, off, len, nPieces, poly, out);
    return cudaGetLastError();
}
template cudaError_t launch_crc_pieces<uint32_t>(const uint8_t*, uint64_t, uint32_t, const uint64_t*, const uint64_t*, uint32_t, uint32_t, uint32_t*, cudaStream_t);
template cudaError_t launch_crc_pieces<uint64_t>(const uint8_t*, uint64_t, uint32_t, const uint64_t*, const uint64_t*, uint32_t, uint64_t, uint64_t*, cudaStream_t);

template <typename T> static int crc_device(b200z_ctx* ctx, const void* d_src, size_t n, T poly, T* result) {
    if (!ctx || !result || (!d_src && n)) return B200Z_E_PARAM;
    *result = 0;
    if (!n) return 0;
    CU(cudaSetDevice(ctx->device));
    const uint32_t nPieces = (uint32_t)((n + (1ull << B2Z_CRC_PIECE_LOG) - 1) >> B2Z_CRC_PIECE_LOG);
    if (ctx->cks.reserve((size_t)nPieces * sizeof(T) + 64)) return fail(ctx, B200Z_E_MEMORY, "device scratch allocation failed%s");
    CU(launch_crc_pieces<T>((const uint8_t*)d_src, n, B2Z_CRC_PIECE_LOG, nullptr, nullptr, nPieces, poly, (T*)ctx->cks.p, ctx->stream));
    std::vector<T> pieces(nPieces);
    CU(cudaMemcpyAsync(pieces.data(), ctx->cks.p, (size_t)nPieces * sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 1;
    *result = crc_fold<T>(pieces, n, B2Z_CRC_PIECE_LOG, poly);
    return 0;
}
#endif

}  // namespace b2z

#ifndef B2Z_CUEMU
extern "C" {

int b200z_crc32_device(b200z_ctx* ctx, const void* d_src, size_t n, uint32_t* crc) { return b2z::crc_device<uint32_t>(ctx, d_src, n, B2Z_CRC32_POLY, crc); }
int b200z_crc64_device(b200z_ctx* ctx, const void* d_src, size_t n, uint64_t* crc) { return b2z::crc_device<uint64_t>(ctx, d_src, n, B2Z_CRC64_POLY, crc); }

static int crc_host_upload(b200z_ctx* ctx, const void* src, size_t n) {
    if (!ctx || (!src && n)) return B200Z_E_PARAM;
    CU(cudaSetDevice(ctx->device));
    if (ctx->dIn.reserve(n + 64)) return fail(ctx, B200Z_E_MEMORY, "device staging allocation failed%s");
    if (n) { CU(cudaMemcpyAsync(ctx->dIn.p, src, n, cudaMemcpyHostToDevice, ctx->stream)); ctx->stat[B200Z_S_H2D_BYTES] += (double)n; }
    return 0;
}
int b200z_crc32_host(b200z_ctx* ctx, const void* src, size_t n, uint32_t* crc) {
    int rc = crc_host_upload(ctx, src, n); if (rc) return rc;
    return b200z_crc32_device(ctx, ctx->dIn.p, n, crc);
}
int b200z_crc64_host(b200z_ctx* ctx, const void* src, size_t n, uint64_t* crc) {
    int rc = crc_host_upload(ctx, src, n); if (rc) return rc;
    return b200z_crc64_device(ctx, ctx->dIn.p, n, crc);
}
// host-only helper of the same arithmetic (no device needed): crc(A || B) from crc(A), crc(B), |B|
uint32_t b200z_crc32_combine(uint32_t crcA, uint32_t crcB, uint64_t lenB) { return b2z::gf_mul<uint32_t>(crcA, b2z::gf_xpow8<uint32_t>(lenB, B2Z_CRC32_POLY), B2Z_CRC32_POLY) ^ crcB; }
uint64_t b200z_crc64_combine(uint64_t crcA, uint64_t crcB, uint64_t lenB) { return b2z::gf_mul<uint64_t>(crcA, b2z::gf_xpow8<uint64_t>(lenB, B2Z_CRC64_POLY), B2Z_CRC64_POLY) ^ crcB; }

}  // extern "C"
#endif
