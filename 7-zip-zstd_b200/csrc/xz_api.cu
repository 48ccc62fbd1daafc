// xz_api.cu -- the .xz container around the GPU LZMA2 coder (SURVEY.md 8(f) item 2): what XzEncoder.cpp / XzDecoder.cpp + C/XzEnc.c,
// C/XzDec.c, C/Xz.c do around Lzma2Enc / Lzma2Dec.  Host code only in this file; the payload is coded by lzma2_enc.cu /
// lzma2_parse.cu / lzma2_dec.cu and the block checks are computed by b2z_crc.cu.
//
//   writer   every dictionary-reset block of the encoder's chunk stream (= one 2^frameLog-byte frame) becomes one xz Block with both
//            sizes in its header, so that any multi-threaded xz decoder -- and ours -- can decode the Blocks independently
//            (the layout `xz -T` / XzEnc.c:1236 Xz_Encode with blockSize write).  Check: none, CRC32 or CRC64 (7-Zip's default, Xz.h:34).
//   reader   Stream Header / Blocks / Index / Footer are parsed and verified on the host (CRC32 of the small fields); the Blocks'
//            LZMA2 payloads are spliced into one chunk stream for the GPU decoder (their end markers dropped), the Block checks
//            are verified on the decoded bytes while they are still in HBM (CRC32, CRC64, SHA-256).
//            Filters in front of LZMA2 -- Delta, x86, PowerPC, ARM, ARM-Thumb, SPARC, ARM64, RISC-V -- are undone on the GPU
//            (b2z_filter.cu) per Block; IA64 chains are B200Z_E_UNSUPPORTED.
// Format: https://tukaani.org/xz/xz-file-format.txt as implemented by C/Xz.c, C/XzEnc.c:150-330 (headers, index, footer), C/XzDec.c:1126-1600.
#include <vector>
#include "b2z_ctx.h"
#include "b2z_lzma2.h"
#include "b2z_kernels.h"

namespace {

// 7-Zip method id of a filter -> xz Filter ID (xz-file-format 5.3); 0 = not a filter the writer knows
uint32_t xz_filter_id(uint32_t methodId) {
    switch (methodId) {
    case 0x03u: return 0x03u; case 0x03030103u: return 0x04u; case 0x03030205u: return 0x05u; case 0x03030501u: return 0x07u;
    case 0x03030701u: return 0x08u; case 0x03030805u: return 0x09u; case 0x0Au: return 0x0Au; case 0x0Bu: return 0x0Bu; default: return 0u;
    }
}

const uint8_t kMagic[6] = { 0xFD, '7', 'z', 'X', 'Z', 0x00 };
const uint8_t kFooterMagic[2] = { 'Y', 'Z' };

uint32_t crc32_small(const uint8_t* p, size_t n) {               // container fields only (a few bytes each)
    uint32_t c = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; i++) { c ^= p[i]; for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1u))); }
    return ~c;
}
void put32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24); }
uint32_t get32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
size_t put_vli(uint8_t* p, uint64_t v) { size_t n = 0; while (v >= 0x80) { p[n++] = (uint8_t)(v | 0x80); v >>= 7; } p[n++] = (uint8_t)v; return n; }
// -> bytes consumed, 0 on error
size_t get_vli(const uint8_t* p, size_t avail, uint64_t* v) {
    uint64_t r = 0;
    for (size_t i = 0; i < 9 && i < avail; i++) {
        r |= (uint64_t)(p[i] & 0x7F) << (7 * i);
        if (!(p[i] & 0x80)) { if (p[i] == 0 && i) return 0; *v = r; return i + 1; }
    }
    return 0;
}
uint32_t check_bytes(uint32_t type) { return type == 0 ? 0u : (type <= 3 ? 4u : (type <= 6 ? 8u : (type <= 9 ? 16u : (type <= 12 ? 32u : 64u)))); }

struct Cut { uint64_t srcOff, srcEnd, dstSize; };
struct CutEmit {                                                   // fills a caller-sized array (lzma2_walk is host + device code)
    Cut* out; uint32_t cap;
    __host__ __device__ void operator()(uint32_t i, uint64_t srcOff, uint64_t srcEnd, uint64_t, uint64_t dstSize) const {
        if (i < cap) { out[i].srcOff = srcOff; out[i].srcEnd = srcEnd; out[i].dstSize = dstSize; }
    }
};
// the dictionary-reset blocks of a chunk stream (two header walks: count, then fill)
uint32_t walk_cuts(const uint8_t* lz, size_t n, std::vector<Cut>& cuts, b2z::Lz2Counts& c) {
    b2z::lzma2_walk(lz, n, c, CutEmit{ nullptr, 0 });
    cuts.assign(c.nBlocks, Cut{ 0, 0, 0 });
    if (c.nBlocks) b2z::lzma2_walk(lz, n, c, CutEmit{ cuts.data(), c.nBlocks });
    return c.status;
}

}  // namespace

extern "C" {

size_t b200z_xz_wrap_bound(size_t lzma2Size, uint32_t nBlocks) { return lzma2Size + (size_t)nBlocks * 72u + 64u; }

// Host only.  lzma2 = a chunk stream (... 0x00) whose dictionary resets delimit the Blocks; checks[i] = the check value of Block i's
// uncompressed bytes (ignored for checkType 0).  checkType: 0 none, 1 CRC32, 4 CRC64.  filterId != 0: every Block declares that
// filter (7-Zip method id; prop = delta distance / start offset) in front of LZMA2 -- the payload must have been filtered per Block.
int b200z_xz_wrap(const void* lzma2v, size_t lzma2Size, uint32_t dictProp, uint32_t checkType, const uint64_t* checks, uint32_t nChecks,
                  uint32_t filterId, uint32_t filterProp, void* dstv, size_t cap, size_t* out) {
    if (!lzma2v || !dstv || !out || (checkType != 0 && checkType != 1 && checkType != 4) || dictProp > 40) return B200Z_E_PARAM;
    if (filterId && (!xz_filter_id(filterId) || (filterId == 0x03u && (filterProp < 1 || filterProp > 256)))) return B200Z_E_PARAM;
    const uint8_t* lz = (const uint8_t*)lzma2v; uint8_t* dst = (uint8_t*)dstv;
    std::vector<Cut> cuts;
    b2z::Lz2Counts c;
    if (walk_cuts(lz, lzma2Size, cuts, c)) return B200Z_E_CORRUPT;
    if (checkType && nChecks < cuts.size()) return B200Z_E_PARAM;
    if (cap < b200z_xz_wrap_bound(lzma2Size, (uint32_t)cuts.size())) return B200Z_E_DSTSIZE;
    const uint32_t cb = check_bytes(checkType);
    size_t o = 0;
    memcpy(dst, kMagic, 6); dst[6] = 0; dst[7] = (uint8_t)checkType; put32(dst + 8, crc32_small(dst + 6, 2)); o = 12;
    std::vector<uint8_t> index; index.push_back(0);
    { uint8_t t[10]; const size_t k = put_vli(t, cuts.size()); index.insert(index.end(), t, t + k); }
    for (size_t b = 0; b < cuts.size(); b++) {
        const uint64_t pack = cuts[b].srcEnd - cuts[b].srcOff + 1;   // + this Block's own end marker
        uint8_t h[64]; size_t k = 1;
        h[k++] = (uint8_t)(0xC0 | (filterId ? 1 : 0));              // one or two filters; compressed and uncompressed size present
        k += put_vli(h + k, pack); k += put_vli(h + k, cuts[b].dstSize);
        if (filterId == 0x03u) { h[k++] = 0x03; h[k++] = 1; h[k++] = (uint8_t)(filterProp - 1u); }
        else if (filterId) { h[k++] = (uint8_t)xz_filter_id(filterId); h[k++] = filterProp ? 4 : 0; if (filterProp) { put32(h + k, filterProp); k += 4; } }
        h[k++] = 0x21; h[k++] = 1; h[k++] = (uint8_t)dictProp;      // LZMA2, one property byte
        while ((k + 4) & 3) h[k++] = 0;
        h[0] = (uint8_t)((k + 4) / 4 - 1);
        put32(h + k, crc32_small(h, k)); k += 4;
        memcpy(dst + o, h, k); o += k;
        memcpy(dst + o, lz + cuts[b].srcOff, (size_t)(pack - 1)); o += (size_t)(pack - 1); dst[o++] = 0;
        for (uint64_t pad = pack; pad & 3; pad++) dst[o++] = 0;
        for (uint32_t i = 0; i < cb; i++) dst[o++] = (uint8_t)(checks[b] >> (8 * i));
        uint8_t t[20]; size_t tk = put_vli(t, k + pack + cb); tk += put_vli(t + tk, cuts[b].dstSize);
        index.insert(index.end(), t, t + tk);
    }
    while (index.size() & 3) index.push_back(0);
    { uint8_t t[4]; put32(t, crc32_small(index.data(), index.size())); index.insert(index.end(), t, t + 4); }
    memcpy(dst + o, index.data(), index.size()); o += index.size();
    uint8_t f[12];
    put32(f + 4, (uint32_t)(index.size() / 4 - 1)); f[8] = 0; f[9] = (uint8_t)checkType; put32(f, crc32_small(f + 4, 6)); f[10] = kFooterMagic[0]; f[11] = kFooterMagic[1];
    memcpy(dst + o, f, 12); o += 12;
    *out = o;
    return 0;
}

// Host only: the Blocks of every Stream in src (concatenated Streams and Stream Padding allowed), container fields verified.
int b200z_xz_parse(const void* srcv, size_t n, b200z_xz_block* blocks, uint32_t cap, uint32_t* nBlocks, uint64_t* total) {
    if (!srcv || !nBlocks) return B200Z_E_PARAM;
    const uint8_t* s = (const uint8_t*)srcv;
    size_t ip = 0; uint32_t nb = 0; uint64_t tot = 0; bool any = false;
    while (ip < n) {
        if (any) { size_t z = ip; while (z < n && s[z] == 0) z++; if (z == n) break; if ((z - ip) & 3) return B200Z_E_CORRUPT; ip = z; }   // Stream Padding
        if (n - ip < 12 || memcmp(s + ip, kMagic, 6) || s[ip + 6] != 0 || (s[ip + 7] & 0xF0) || get32(s + ip + 8) != crc32_small(s + ip + 6, 2)) return B200Z_E_CORRUPT;
        const uint32_t checkType = s[ip + 7], cb = check_bytes(checkType);
        const size_t streamStart = ip; ip += 12;
        const uint32_t firstBlock = nb;
        std::vector<std::pair<uint64_t, uint64_t>> recs;           // (unpadded size, uncompressed size) as read from the Blocks
        while (ip < n && s[ip] != 0) {                              // Block (Index Indicator is 0x00)
            const size_t hs = ((size_t)s[ip] + 1) * 4;
            if (n - ip < hs || get32(s + ip + hs - 4) != crc32_small(s + ip, hs - 4)) return B200Z_E_CORRUPT;
            const uint8_t fl = s[ip + 1];
            if (fl & 0x3C) return B200Z_E_UNSUPPORTED;
            size_t k = 2; uint64_t pack = ~0ull, unpack = ~0ull; size_t m;
            if (fl & 0x40) { m = get_vli(s + ip + k, hs - 4 - k, &pack); if (!m) return B200Z_E_CORRUPT; k += m; }
            if (fl & 0x80) { m = get_vli(s + ip + k, hs - 4 - k, &unpack); if (!m) return B200Z_E_CORRUPT; k += m; }
            // List of Filter Flags: up to three filters in front of LZMA2, which must come last (xz-file-format 3.1.3 / Xz.h:68 XZ_NUM_FILTERS_MAX).
            // Kept as 7-Zip method ids + one property each, for b200z_filter_device: Delta 0x03 (distance), x86 0x04, PowerPC 0x05, ARM 0x07,
            // ARM-Thumb 0x08, SPARC 0x09, ARM64 0x0A, RISC-V 0x0B (start offset); IA64 0x06 is not built -> unsupported
            const uint32_t nf = (fl & 3u) + 1u;
            uint32_t fId[3] = { 0, 0, 0 }, fProp[3] = { 0, 0, 0 }, dictProp = 0;
            for (uint32_t f = 0; f < nf; f++) {
                uint64_t id, psz;
                m = get_vli(s + ip + k, hs - 4 - k, &id); if (!m) return B200Z_E_CORRUPT; k += m;
                m = get_vli(s + ip + k, hs - 4 - k, &psz); if (!m || k + m + psz > hs - 4) return B200Z_E_CORRUPT; k += m;
                if (f + 1 == nf) {
                    if (id != 0x21) return (id == 0x03 || (id >= 0x04 && id <= 0x0B)) ? B200Z_E_CORRUPT : B200Z_E_UNSUPPORTED;   // a filter that cannot be last / not LZMA2
                    if (psz != 1) return B200Z_E_CORRUPT;
                    dictProp = s[ip + k];
                } else if (id == 0x03) {
                    if (psz != 1) return B200Z_E_CORRUPT;
                    fId[f] = 0x03u; fProp[f] = (uint32_t)s[ip + k] + 1u;
                } else if (id == 0x04 || id == 0x05 || id == 0x07 || id == 0x08 || id == 0x09 || id == 0x0A || id == 0x0B) {
                    if (psz != 0 && psz != 4) return B200Z_E_CORRUPT;
                    fId[f] = id == 0x04 ? 0x03030103u : (id == 0x05 ? 0x03030205u : (id == 0x07 ? 0x03030501u : (id == 0x08 ? 0x03030701u : (id == 0x09 ? 0x03030805u : (uint32_t)id))));
                    fProp[f] = psz ? get32(s + ip + k) : 0u;
                    if (id != 0x04 && (fProp[f] & (id == 0x08 || id == 0x0B ? 1u : 3u))) return B200Z_E_UNSUPPORTED;      // BranchMisc.cpp:99, XzDec.c:124
                } else return B200Z_E_UNSUPPORTED;                  // 0x21 in front, IA64, unknown ids
                k += (size_t)psz;
            }
            if (dictProp > 40) return B200Z_E_CORRUPT;
            for (; k < hs - 4; k++) if (s[ip + k]) return B200Z_E_CORRUPT;
            const size_t dataOff = ip + hs;
            {   // every Block's payload is walked chunk header by chunk header, declared sizes or not: it must be ONE complete LZMA2 stream --
                // first chunk a dictionary reset, end marker exactly where the Compressed Size says, chunk sizes adding up to the
                // Uncompressed Size -- which is what XzDec / liblzma enforce by decoding Block by Block (C/XzDec.c:1100-1300)
                b2z::Lz2Counts c;
                const size_t avail = (pack != ~0ull && pack < n - dataOff) ? (size_t)pack : n - dataOff;
                b2z::lzma2_walk(s + dataOff, avail, c, CutEmit{ nullptr, 0 });
                if (c.status) return B200Z_E_CORRUPT;
                if (pack != ~0ull && pack != c.srcUsed) return B200Z_E_CORRUPT;
                if (unpack != ~0ull && unpack != c.total) return B200Z_E_CORRUPT;
                pack = c.srcUsed; unpack = c.total;
            }
            const size_t padded = (size_t)((pack + 3) & ~3ull);
            if (pack == 0 || n - dataOff < padded + cb) return B200Z_E_CORRUPT;
            for (size_t z = (size_t)pack; z < padded; z++) if (s[dataOff + z]) return B200Z_E_CORRUPT;
            if (blocks && nb < cap) {
                b200z_xz_block& B = blocks[nb];
                B.packOff = dataOff; B.packSize = pack; B.unpackSize = unpack; B.dictProp = dictProp; B.checkType = checkType; B.check = 0;
                B.nFilters = nf - 1u; for (uint32_t f = 0; f < 3; f++) { B.filterId[f] = fId[f]; B.filterProp[f] = fProp[f]; }
                for (uint32_t i = 0; i < cb && i < 8; i++) B.check |= (uint64_t)s[dataOff + padded + i] << (8 * i);
            }
            if (tot + unpack < tot) return B200Z_E_CORRUPT;          // (64-bit wrap of the declared sizes)
            nb++; tot += unpack;
            recs.emplace_back((uint64_t)hs + pack + cb, unpack);
            ip = dataOff + padded + cb;
        }
        // Index
        const size_t idx0 = ip; uint64_t cnt = 0; size_t m;
        if (ip >= n) return B200Z_E_CORRUPT;
        ip++; m = get_vli(s + ip, n - ip, &cnt); if (!m || cnt != nb - firstBlock) return B200Z_E_CORRUPT; ip += m;
        for (uint64_t r = 0; r < cnt; r++) {
            uint64_t a, b;
            m = get_vli(s + ip, n - ip, &a); if (!m) return B200Z_E_CORRUPT; ip += m;
            m = get_vli(s + ip, n - ip, &b); if (!m) return B200Z_E_CORRUPT; ip += m;
            if (a != recs[(size_t)r].first || b != recs[(size_t)r].second) return B200Z_E_CORRUPT;
        }
        while ((ip - idx0) & 3) { if (ip >= n || s[ip]) return B200Z_E_CORRUPT; ip++; }
        if (n - ip < 16 || get32(s + ip) != crc32_small(s + idx0, ip - idx0)) return B200Z_E_CORRUPT;
        ip += 4;
        const size_t indexSize = ip - idx0;
        if (get32(s + ip) != crc32_small(s + ip + 4, 6) || ((size_t)get32(s + ip + 4) + 1) * 4 != indexSize || s[ip + 8] != 0 || s[ip + 9] != s[streamStart + 7] ||
            s[ip + 10] != kFooterMagic[0] || s[ip + 11] != kFooterMagic[1]) return B200Z_E_CORRUPT;
        ip += 12; any = true;
    }
    if (!any) return B200Z_E_CORRUPT;
    *nBlocks = nb; if (total) *total = tot;
    return (blocks && nb > cap) ? B200Z_E_DSTSIZE : 0;
}

size_t b200z_xz_compress_bound(b200z_ctx* ctx, size_t n) {
    const size_t lz = b200z_lzma2_compress_bound(ctx, n);
    const uint32_t fl = ctx ? ctx->geom.frameLog : B2Z_DEF_FRAMELOG;
    return b200z_xz_wrap_bound(lz, (uint32_t)((n >> fl) + 1));
}

// XzEncoder.cpp:  .xz with one Block per 2^FRAMELOG input bytes; checkType 0 none, 1 CRC32, 4 CRC64.  filterId != 0: that filter
// (Delta 0x03, x86 0x03030103, PowerPC, ARM, ARM Thumb, SPARC, ARM64, RISC-V 0x0B; 7-Zip method ids) runs on the GPU in front of
// LZMA2, Block by Block
int b200z_xz_compress_host(b200z_ctx* ctx, const void* src, size_t n, void* dst, size_t cap, size_t* out, uint32_t checkType,
                           uint32_t filterId, uint32_t filterProp) {
    if (!ctx || !out || (!src && n) || !dst) return B200Z_E_PARAM;
    if (checkType != 0 && checkType != 1 && checkType != 4) return fail(ctx, B200Z_E_PARAM, "xz: check type must be 0 (none), 1 (CRC32) or 4 (CRC64)%s");
    if (filterId && !xz_filter_id(filterId)) return fail(ctx, B200Z_E_UNSUPPORTED, "xz: filter not built on the GPU%s");
    { const int prc = lz2_check_props(ctx); if (prc) return prc; }   // lc / lp / pb travel in the chunk headers: no Block Header field for them
    if (cap < b200z_xz_compress_bound(ctx, n)) return fail(ctx, B200Z_E_DSTSIZE, "dstCap < b200z_xz_compress_bound%s");
    CU(cudaSetDevice(ctx->device));
    const size_t lzCap = b200z_lzma2_compress_bound(ctx, n);
    if (ctx->dIn.reserve(n + 64) || ctx->dOut.reserve(lzCap + 64)) return fail(ctx, B200Z_E_MEMORY, "device staging allocation failed%s");
    if (n) { CU(cudaMemcpyAsync(ctx->dIn.p, src, n, cudaMemcpyHostToDevice, ctx->stream)); ctx->stat[B200Z_S_H2D_BYTES] += (double)n; }
    // Block checks first: they cover the ORIGINAL bytes (one piece per frame, while the input is in HBM)
    const uint32_t fl = ctx->geom.frameLog;
    const uint32_t nFrames = (uint32_t)((n + ((size_t)1 << fl) - 1) >> fl);
    std::vector<uint64_t> checks(nFrames ? nFrames : 1, 0);
    if (checkType && nFrames) {
        if (ctx->cks.reserve((size_t)nFrames * 8 + 64)) return fail(ctx, B200Z_E_MEMORY, "device scratch allocation failed%s");
        if (checkType == 1) {
            CU(b2z::launch_crc_pieces<uint32_t>((const uint8_t*)ctx->dIn.p, n, fl, nullptr, nullptr, nFrames, B2Z_CRC32_POLY, (uint32_t*)ctx->cks.p, ctx->stream));
            std::vector<uint32_t> t(nFrames);
            CU(cudaMemcpyAsync(t.data(), ctx->cks.p, (size_t)nFrames * 4, cudaMemcpyDeviceToHost, ctx->stream)); CU(cudaStreamSynchronize(ctx->stream));
            for (uint32_t i = 0; i < nFrames; i++) checks[i] = t[i];
        } else {
            CU(b2z::launch_crc_pieces<uint64_t>((const uint8_t*)ctx->dIn.p, n, fl, nullptr, nullptr, nFrames, B2Z_CRC64_POLY, (uint64_t*)ctx->cks.p, ctx->stream));
            CU(cudaMemcpyAsync(checks.data(), ctx->cks.p, (size_t)nFrames * 8, cudaMemcpyDeviceToHost, ctx->stream)); CU(cudaStreamSynchronize(ctx->stream));
        }
        ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 1;
    }
    int rc;
    if (filterId && n) {                                            // every frame = one Block = one independent run of the filter
        rc = b2z_filter_units_device(ctx, filterId, 1, ctx->dIn.p, n, filterProp, fl);
        if (rc) return rc;
    }
    size_t lzSize = 0; uint32_t prop = 0;
    rc = b200z_lzma2_compress_device(ctx, ctx->dIn.p, n, ctx->dOut.p, lzCap, &lzSize, &prop);
    if (rc) return rc;
    std::vector<uint8_t> lz(lzSize);
    CU(cudaMemcpyAsync(lz.data(), ctx->dOut.p, lzSize, cudaMemcpyDeviceToHost, ctx->stream)); CU(cudaStreamSynchronize(ctx->stream));
    ctx->stat[B200Z_S_D2H_BYTES] += (double)lzSize;
    rc = b200z_xz_wrap(lz.data(), lzSize, prop, checkType, checks.data(), (uint32_t)checks.size(), filterId, filterProp, dst, cap, out);
    return rc ? fail(ctx, rc, "xz: container assembly failed%s") : 0;
}

// XzDecoder.cpp: any .xz whose Blocks are LZMA2-only; Blocks decode in parallel on the GPU; CRC32 / CRC64 checks are verified
int b200z_xz_decompress_host(b200z_ctx* ctx, const void* srcv, size_t n, void* dst, size_t cap, size_t* out) {
    if (!ctx || !out || !srcv || (!dst && cap)) return B200Z_E_PARAM;
    *out = 0;
    const uint8_t* s = (const uint8_t*)srcv;
    uint32_t nb = 0; uint64_t total = 0;
    int rc = b200z_xz_parse(s, n, nullptr, 0, &nb, &total);
    if (rc) return fail(ctx, rc, rc == B200Z_E_UNSUPPORTED ? "xz: filter chain other than a single LZMA2%s" : "xz: malformed container%s");
    if (total > cap) return fail(ctx, B200Z_E_DSTSIZE, "destination too small%s");
    if (!nb) return 0;
    std::vector<b200z_xz_block> blocks(nb);
    rc = b200z_xz_parse(s, n, blocks.data(), nb, &nb, &total);
    if (rc) return fail(ctx, rc, "xz: malformed container%s");
    // splice the Blocks' chunk streams into one (every Block starts with a dictionary reset, xz-file-format 5.3.1 / Lzma2Dec.c:97)
    size_t lzSize = 1; uint32_t prop = 0;
    for (const auto& b : blocks) { lzSize += (size_t)b.packSize - 1; if (b.dictProp > prop) prop = b.dictProp; }
    std::vector<uint8_t> lz(lzSize);
    size_t o = 0;
    for (const auto& b : blocks) {
        if (b.packSize < 1 || s[b.packOff + b.packSize - 1] != 0) return fail(ctx, B200Z_E_CORRUPT, "xz: Block without an end marker%s");
        if (b.packSize > 1 && s[b.packOff] != 0x01 && s[b.packOff] < 0xE0) return fail(ctx, B200Z_E_CORRUPT, "xz: Block does not start with a dictionary reset%s");
        memcpy(lz.data() + o, s + b.packOff, (size_t)b.packSize - 1); o += (size_t)b.packSize - 1;
    }
    lz[o++] = 0;
    size_t got = 0;
    rc = b200z_lzma2_decompress_host(ctx, lz.data(), lzSize, prop, dst, cap, &got);
    if (rc) return rc;
    if (got != total) return fail(ctx, B200Z_E_CORRUPT, "xz: decoded size differs from the Block headers%s");
    // a Block must decode to exactly its declared size: the decoder's dictionary-reset blocks must line up with the xz Blocks
    {
        std::vector<Cut> cuts; b2z::Lz2Counts c;
        walk_cuts(lz.data(), lzSize, cuts, c);
        size_t ci = 0;
        for (const auto& b : blocks) {
            uint64_t acc = 0;
            while (ci < cuts.size() && acc < b.unpackSize) acc += cuts[ci++].dstSize;
            if (acc != b.unpackSize) return fail(ctx, B200Z_E_CORRUPT, "xz: Block size differs from its header%s");
        }
    }
    // Filters in front of LZMA2 (xz --x86, --delta ...): undone per Block, last filter first, on the decoded bytes in HBM; the Block's
    // bytes are then copied to the caller again.  A filter's position counter starts at its start offset in every Block.
    {
        uint64_t pos = 0;
        for (uint32_t i = 0; i < nb; i++) {
            const b200z_xz_block& b = blocks[i];
            if (b.nFilters && b.unpackSize) {
                uint8_t* d = (uint8_t*)ctx->dOut.p + pos;
                const bool staged = ((uintptr_t)d & 3u) != 0;                     // the branch converters want 4-byte (Thumb: 2-byte) alignment
                if (staged) {
                    if (ctx->slots.reserve((size_t)b.unpackSize + 64)) return fail(ctx, B200Z_E_MEMORY, "device scratch allocation failed%s");
                    CU(cudaMemcpyAsync(ctx->slots.p, d, (size_t)b.unpackSize, cudaMemcpyDeviceToDevice, ctx->stream));
                }
                for (int f = (int)b.nFilters - 1; f >= 0; f--) {
                    rc = b200z_filter_device(ctx, b.filterId[f], 0, staged ? ctx->slots.p : (void*)d, (size_t)b.unpackSize, b.filterProp[f]);
                    if (rc) return rc;
                }
                if (staged) CU(cudaMemcpyAsync(d, ctx->slots.p, (size_t)b.unpackSize, cudaMemcpyDeviceToDevice, ctx->stream));
                CU(cudaMemcpyAsync((uint8_t*)dst + pos, d, (size_t)b.unpackSize, cudaMemcpyDeviceToHost, ctx->stream));
                CU(cudaStreamSynchronize(ctx->stream));
            }
            pos += b.unpackSize;
        }
    }
    // Block checks on the decoded bytes, which b200z_lzma2_decompress_host left in the context's output arena (Streams of one file
    // may carry different check types: one kernel launch per type present; unknown types are not verified)
    for (uint32_t type = 1; type <= 4; type += 3) {
        std::vector<uint64_t> off, len; std::vector<uint32_t> which;
        uint64_t pos = 0;
        for (uint32_t i = 0; i < nb; i++) { if (blocks[i].checkType == type) { off.push_back(pos); len.push_back(blocks[i].unpackSize); which.push_back(i); } pos += blocks[i].unpackSize; }
        const uint32_t m = (uint32_t)which.size();
        if (!m) continue;
        if (ctx->batchOff.reserve((size_t)m * 8) || ctx->batchSize.reserve((size_t)m * 8) || ctx->cks.reserve((size_t)m * 8 + 64)) return fail(ctx, B200Z_E_MEMORY, "device scratch allocation failed%s");
        CU(cudaMemcpyAsync(ctx->batchOff.p, off.data(), (size_t)m * 8, cudaMemcpyHostToDevice, ctx->stream));
        CU(cudaMemcpyAsync(ctx->batchSize.p, len.data(), (size_t)m * 8, cudaMemcpyHostToDevice, ctx->stream));
        std::vector<uint64_t> have(m, 0);
        if (type == 1) {
            CU(b2z::launch_crc_pieces<uint32_t>((const uint8_t*)ctx->dOut.p, got, 0, (const uint64_t*)ctx->batchOff.p, (const uint64_t*)ctx->batchSize.p, m, B2Z_CRC32_POLY, (uint32_t*)ctx->cks.p, ctx->stream));
            std::vector<uint32_t> t(m);
            CU(cudaMemcpyAsync(t.data(), ctx->cks.p, (size_t)m * 4, cudaMemcpyDeviceToHost, ctx->stream)); CU(cudaStreamSynchronize(ctx->stream));
            for (uint32_t i = 0; i < m; i++) have[i] = t[i];
        } else {
            CU(b2z::launch_crc_pieces<uint64_t>((const uint8_t*)ctx->dOut.p, got, 0, (const uint64_t*)ctx->batchOff.p, (const uint64_t*)ctx->batchSize.p, m, B2Z_CRC64_POLY, (uint64_t*)ctx->cks.p, ctx->stream));
            CU(cudaMemcpyAsync(have.data(), ctx->cks.p, (size_t)m * 8, cudaMemcpyDeviceToHost, ctx->stream)); CU(cudaStreamSynchronize(ctx->stream));
        }
        ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 1;
        for (uint32_t i = 0; i < m; i++) if (have[i] != blocks[which[i]].check) return fail(ctx, B200Z_E_CHECKSUM, "xz: Block check mismatch%s");
    }
    {   // SHA-256 checks (type 10): one thread per Block on the decoded bytes; the 32 check bytes follow the Block's padded payload
        std::vector<uint64_t> off, len; std::vector<uint32_t> which;
        uint64_t pos = 0;
        for (uint32_t i = 0; i < nb; i++) { if (blocks[i].checkType == 10u) { off.push_back(pos); len.push_back(blocks[i].unpackSize); which.push_back(i); } pos += blocks[i].unpackSize; }
        const uint32_t m = (uint32_t)which.size();
        if (m) {
            if (ctx->batchOff.reserve((size_t)m * 8) || ctx->batchSize.reserve((size_t)m * 8) || ctx->cks.reserve((size_t)m * 32 + 64)) return fail(ctx, B200Z_E_MEMORY, "device scratch allocation failed%s");
            CU(cudaMemcpyAsync(ctx->batchOff.p, off.data(), (size_t)m * 8, cudaMemcpyHostToDevice, ctx->stream));
            CU(cudaMemcpyAsync(ctx->batchSize.p, len.data(), (size_t)m * 8, cudaMemcpyHostToDevice, ctx->stream));
            CU(b2z::launch_sha256_pieces((const uint8_t*)ctx->dOut.p, (const uint64_t*)ctx->batchOff.p, (const uint64_t*)ctx->batchSize.p, m, (uint32_t*)ctx->cks.p, ctx->stream));
            std::vector<uint32_t> have((size_t)m * 8);
            CU(cudaMemcpyAsync(have.data(), ctx->cks.p, (size_t)m * 32, cudaMemcpyDeviceToHost, ctx->stream)); CU(cudaStreamSynchronize(ctx->stream));
            ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 1;
            for (uint32_t i = 0; i < m; i++) {
                const b200z_xz_block& b = blocks[which[i]];
                const uint8_t* want = s + b.packOff + ((b.packSize + 3) & ~3ull);
                for (uint32_t k = 0; k < 8; k++)
                    if (have[(size_t)i * 8 + k] != (((uint32_t)want[4 * k] << 24) | ((uint32_t)want[4 * k + 1] << 16) | ((uint32_t)want[4 * k + 2] << 8) | want[4 * k + 3]))
                        return fail(ctx, B200Z_E_CHECKSUM, "xz: Block check (SHA-256) mismatch%s");
            }
        }
    }
    *out = got;
    return 0;
}

}  // extern "C"
