// coder_props.cpp -- drives the LZMA2 / FLZMA2 encoders of libb200z_7z.so with the literal / position context bits
// (kLitContextBits, kLitPosBits, kPosStateBits) as 7-Zip's -m0=lzma2:lc=N:lp=N:pb=N sends them (SetCoderProperties, then Code()).
// usage: coder_props <lib.so> <input file> <packed output prefix> lc lp pb      (needs a GPU)
//        coder_props <lib.so> --props                                            (property checks only, no GPU)
// Writes <prefix>.lzma2 / <prefix>.flzma2 (raw LZMA2 streams); the caller checks their chunk headers and decodes them.
#include <dlfcn.h>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>
#include "../../7-zip-zstd_b200/codec/b2z_7zip_abi.h"

struct MemIn final : ISequentialInStream {
    const std::vector<Byte>& d; size_t pos = 0; UInt32 refs = 1;
    explicit MemIn(const std::vector<Byte>& v) : d(v) {}
    HRESULT QueryInterface(const GUID&, void** o) override { *o = nullptr; return E_NOINTERFACE; }
    UInt32 AddRef() override { return ++refs; }
    UInt32 Release() override { return --refs; }
    HRESULT Read(void* data, UInt32 size, UInt32* processed) override {
        size_t n = d.size() - pos; if (n > size) n = size;
        memcpy(data, d.data() + pos, n); pos += n; if (processed) *processed = (UInt32)n; return S_OK;
    }
};
struct MemOut final : ISequentialOutStream {
    std::vector<Byte> d; UInt32 refs = 1;
    HRESULT QueryInterface(const GUID&, void** o) override { *o = nullptr; return E_NOINTERFACE; }
    UInt32 AddRef() override { return ++refs; }
    UInt32 Release() override { return --refs; }
    HRESULT Write(const void* data, UInt32 size, UInt32* processed) override {
        d.insert(d.end(), (const Byte*)data, (const Byte*)data + size); if (processed) *processed = size; return S_OK;
    }
};

#define CHECK(c) do { if (!(c)) { fprintf(stderr, "FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

typedef HRESULT (*CreateFn)(UInt32, const GUID*, void**);

// SetCoderProperties with kLitContextBits / kLitPosBits / kPosStateBits (a negative value: not sent) -> its HRESULT
static HRESULT set_props(ICompressSetCoderProperties* s, int lc, int lp, int pb) {
    PROPID ids[4]; PROPVARIANT pv[4]; memset(pv, 0, sizeof(pv)); UInt32 n = 0;
    ids[n] = NCoderPropID::kDictionarySize; pv[n].vt = VT_UI4; pv[n].ulVal = 1u << 20; n++;
    if (lc >= 0) { ids[n] = NCoderPropID::kLitContextBits; pv[n].vt = VT_UI4; pv[n].ulVal = (UInt32)lc; n++; }
    if (lp >= 0) { ids[n] = NCoderPropID::kLitPosBits; pv[n].vt = VT_UI4; pv[n].ulVal = (UInt32)lp; n++; }
    if (pb >= 0) { ids[n] = NCoderPropID::kPosStateBits; pv[n].vt = VT_UI4; pv[n].ulVal = (UInt32)pb; n++; }
    return s->SetCoderProperties(ids, pv, n);
}

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    void* h = dlopen(argv[1], RTLD_NOW);
    if (!h) { fprintf(stderr, "dlopen: %s\n", dlerror()); return 1; }
    auto CreateEncoder = (CreateFn)dlsym(h, "CreateEncoder");
    CHECK(CreateEncoder);
    const GUID iidCoder = b2z_iid(4, kIID_Coder);
    const bool run = std::string(argv[2]) != "--props";
    if (run) CHECK(argc >= 7);
    std::vector<Byte> input;
    if (run) { FILE* f = fopen(argv[2], "rb"); CHECK(f); Byte buf[1 << 16]; size_t k; while ((k = fread(buf, 1, sizeof(buf), f)) > 0) input.insert(input.end(), buf, buf + k); fclose(f); }
    for (UInt32 idx = 1; idx <= 2; idx++) {                              // 1 LZMA2, 2 FLZMA2
        void* o = nullptr; CHECK(CreateEncoder(idx, &iidCoder, &o) == S_OK && o);
        ICompressCoder* e = (ICompressCoder*)o; ICompressSetCoderProperties* s = nullptr;
        CHECK(e->QueryInterface(b2z_iid(4, kIID_SetProps), (void**)&s) == S_OK);
        // Lzma2Enc_SetProps / FL2_CCtx_setParameter refuse these: E_INVALIDARG
        CHECK(set_props(s, 3, 2, -1) == E_INVALIDARG);                  // lc + lp = 5
        CHECK(set_props(s, -1, 3, -1) == E_INVALIDARG);                 // the engine's lc2 + lp3
        CHECK(set_props(s, 0, 0, 5) == E_INVALIDARG);                   // pb 5
        CHECK(set_props(s, -1, 5, -1) == E_INVALIDARG);                 // lp 5
        CHECK(set_props(s, 9, -1, -1) == E_INVALIDARG);                 // lc 9
        CHECK(set_props(s, 4, 0, 4) == S_OK && set_props(s, 0, 4, 0) == S_OK && set_props(s, -1, 2, -1) == S_OK);
        if (run) {
            CHECK(set_props(s, atoi(argv[4]), atoi(argv[5]), atoi(argv[6])) == S_OK);
            MemIn in(input); MemOut packed;
            const HRESULT r = e->Code(&in, &packed, nullptr, nullptr, nullptr);
            if (r != S_OK) { fprintf(stderr, "encoder %u Code() = 0x%08x\n", (unsigned)idx, (unsigned)r); return 1; }
            CHECK(!packed.d.empty() && packed.d.back() == 0);
            const std::string path = std::string(argv[3]) + (idx == 1 ? ".lzma2" : ".flzma2");
            FILE* f = fopen(path.c_str(), "wb"); CHECK(f); fwrite(packed.d.data(), 1, packed.d.size(), f); fclose(f);
        }
        s->Release(); CHECK(e->Release() == 0);
    }
    printf("coder props ok\n");
    return 0;
}
