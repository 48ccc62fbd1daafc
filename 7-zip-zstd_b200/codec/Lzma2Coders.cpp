// Lzma2Coders.cpp -- NCompress::NLzma2::CEncoder / CFastEncoder / CDecoder for method 21 on top of the b200z C ABI.
// Host-side mirror of the reference wrappers:
//   CPP/7zip/Compress/Lzma2Encoder.{h,cpp}  (SetLzma2Prop :42-77, SetCoderProperties :80-91, WriteCoderProperties :117-121,
//                                            Code :124-150; CFastEncoder :178-364: algo > 3 rejected, block size -> reset interval,
//                                            1-byte property)
//   CPP/7zip/Compress/Lzma2Decoder.{h,cpp}  (SetDecoderProperties2 :40-48 size 1 / <= 40 else E_NOTIMPL, SetFinishMode :51-55,
//                                            Code :95-186, GetInStreamProcessedSize :189-193)
// Same interface sets, property meaning and HRESULT mapping.  Below them: the encoder cuts the input into independent
// dictionary-reset blocks (B200Z_P_FRAMELOG, taken from kBlockSize / kDictionarySize when given) and codes them on the GPU;
// the decoder hands the whole packed stream of a folder to the GPU, which decodes its dictionary-reset blocks in parallel
// (the unit Lzma2DecMt.c:237 uses).
#include "b2z_coder_common.h"

namespace {

int log2_floor(uint64_t v) { int r = 0; while (v >>= 1) r++; return r; }

class CLzma2Encoder final : public ICompressCoder, public ICompressSetCoderProperties, public ICompressSetCoderPropertiesOpt,
                            public ICompressWriteCoderProperties, CoderBase {
    std::atomic<UInt32> refs_{0};
    const bool fast_;
    int frameLog_ = 20;                                        // 1 MiB blocks: thousands of independent blocks per GiB
    int level_ = -1, algo_ = -1;                               // kLevel / kAlgorithm as given (-1: not given)
    int lc_ = -1, lp_ = -1, pb_ = -1;                          // kLitContextBits / kLitPosBits / kPosStateBits (-1: the engine's 2 / 0 / 2)
    PinnedBuf in_, out_;
public:
    UInt64 processedIn = 0, processedOut = 0;
    explicit CLzma2Encoder(bool fast) : fast_(fast) {}
    HRESULT QueryInterface(const GUID& iid, void** out) override {
        *out = nullptr;
        if (iid == kIID_IUnknown || iid == b2z_iid(4, kIID_Coder)) *out = static_cast<ICompressCoder*>(this);
        else if (iid == b2z_iid(4, kIID_SetProps)) *out = static_cast<ICompressSetCoderProperties*>(this);
        else if (iid == b2z_iid(4, kIID_SetPropsOpt) && !fast_) *out = static_cast<ICompressSetCoderPropertiesOpt*>(this);   // CFastEncoder has no Opt interface
        else if (iid == b2z_iid(4, kIID_WriteProps)) *out = static_cast<ICompressWriteCoderProperties*>(this);
        else return E_NOINTERFACE;
        ++refs_; return S_OK;
    }
    UInt32 AddRef() override { return ++refs_; }
    UInt32 Release() override { UInt32 r = --refs_; if (!r) delete this; return r; }

    HRESULT SetCoderProperties(const PROPID* ids, const PROPVARIANT* pv, UInt32 n) override {
        uint64_t blockSize = 0, dictSize = 0;
        int lc = -1, lp = -1, pb = -1;                         // every call starts from the defaults, as Lzma2EncProps_Init does
        for (UInt32 i = 0; i < n; i++) {
            const PROPVARIANT& p = pv[i];
            switch (ids[i]) {
            case NCoderPropID::kBlockSize:                     // Lzma2Encoder.cpp:46-55
                if (p.vt == VT_UI4) blockSize = p.ulVal; else if (p.vt == VT_UI8) blockSize = p.uhVal; else return E_INVALIDARG;
                break;
            case NCoderPropID::kNumThreads: if (p.vt != VT_UI4) return E_INVALIDARG; break;
            case NCoderPropID::kNumThreadGroups: if (p.vt != VT_UI4 || p.ulVal >= (1u << 16)) return E_INVALIDARG; break;
            case NCoderPropID::kDictionarySize: if (p.vt != VT_UI4 && p.vt != VT_UI8) return E_INVALIDARG; dictSize = p.vt == VT_UI4 ? p.ulVal : p.uhVal; break;
            case NCoderPropID::kAlgorithm: if (p.vt != VT_UI4) return E_INVALIDARG; if (fast_ && p.ulVal > 3) return E_INVALIDARG;      // Lzma2Encoder.cpp:197-199
                algo_ = (int)p.ulVal; break;
            case NCoderPropID::kLevel: if (p.vt != VT_UI4) return E_INVALIDARG; level_ = (int)p.ulVal; break;
            // LzmaEnc_SetProps (LzmaEnc.c:541): lc <= 8, lp <= 4, pb <= 4; fast-lzma2 (fl2_compress.c:720-737): lc <= 4
            case NCoderPropID::kLitContextBits: if (p.vt != VT_UI4 || p.ulVal > (fast_ ? 4u : 8u)) return E_INVALIDARG; lc = (int)p.ulVal; break;
            case NCoderPropID::kLitPosBits: if (p.vt != VT_UI4 || p.ulVal > 4) return E_INVALIDARG; lp = (int)p.ulVal; break;
            case NCoderPropID::kPosStateBits: if (p.vt != VT_UI4 || p.ulVal > 4) return E_INVALIDARG; pb = (int)p.ulVal; break;
            case NCoderPropID::kNumFastBytes: case NCoderPropID::kMatchFinderCycles:
                if (p.vt != VT_UI4) return E_INVALIDARG;      // accepted; the GPU coder runs its own finder
                break;
            default: break;                                    // kMatchFinder, kEndMarker, kReduceSize, kAffinity ...: accepted
            }
        }
        // LZMA2 keeps lc + lp <= 4 (Lzma2Enc_SetProps, Lzma2Enc.c:471; fast-lzma2 lclpMax_exceeded); a property not given is the engine's
        if ((lc < 0 ? 2 : lc) + (lp < 0 ? 0 : lp) > 4) return E_INVALIDARG;
        lc_ = lc; lp_ = lp; pb_ = pb;
        // independent block = dictionary = frame: the explicit block size wins, else the dictionary size, else 1 MiB
        const uint64_t want = (blockSize && blockSize != ~0ull) ? blockSize : dictSize;
        if (want) { int fl = log2_floor(want); frameLog_ = fl < 17 ? 17 : (fl > 24 ? 24 : fl); }
        return S_OK;
    }
    // Which parse the level / algorithm asks for, as the reference resolves them: the stock encoder parses by price when
    // algo != 0, algo defaulting to (level < 5 ? 0 : 1) (LzmaEnc.c:97, :570 fastMode); fast-lzma2's strategy is the given
    // algorithm, else its level table's: fast at levels 1-2, opt/ultra from 3 (fl2_compress.c:72-84).  No level given: 5.
    int price_parse() const {
        const int level = level_ < 0 ? 5 : level_;
        if (algo_ >= 0) return algo_ != 0;
        return fast_ ? level >= 3 : level >= 5;
    }
    HRESULT SetCoderPropertiesOpt(const PROPID*, const PROPVARIANT*, UInt32) override { return S_OK; }   // kExpectedDataSize
    HRESULT WriteCoderProperties(ISequentialOutStream* out) override {
        const Byte prop = (Byte)((frameLog_ - 12) * 2);        // dictionary size 2^frameLog (Lzma2Enc_WriteProperties, Lzma2Enc.c:671-690)
        return write_stream(out, &prop, 1);
    }

    HRESULT Code(ISequentialInStream* inS, ISequentialOutStream* outS, const UInt64*, const UInt64*, ICompressProgressInfo* progress) override {
        processedIn = processedOut = 0;
        HRESULT hr = ensure_ctx(); if (hr != S_OK) return hr;
        b200z_set_param(ctx, B200Z_P_FRAMELOG, frameLog_);
        b200z_set_param(ctx, B200Z_P_WINDOWLOG, frameLog_);
        b200z_set_param(ctx, B200Z_P_LZMA2_PARSE, price_parse());
        b200z_set_param(ctx, B200Z_P_LZMA2_LC, lc_ < 0 ? 2 : lc_);
        b200z_set_param(ctx, B200Z_P_LZMA2_LP, lp_ < 0 ? 0 : lp_);
        b200z_set_param(ctx, B200Z_P_LZMA2_PB, pb_ < 0 ? 2 : pb_);
        const size_t batch = (size_t)1 << 30;                  // 1 GiB of input per GPU pass (about a thousand blocks)
        if (!in_.reserve(batch) || !out_.reserve(b200z_lzma2_compress_bound(ctx, batch))) return E_OUTOFMEMORY;
        for (;;) {
            size_t got = batch;
            hr = read_stream(inS, in_.p, &got);
            if (hr != S_OK) return hr;
            if (got == 0) break;
            size_t produced = 0; uint32_t prop = 0;
            int rc = b200z_lzma2_compress_host(ctx, in_.p, got, out_.p, out_.cap, &produced, &prop);
            if (rc) return hr_from_b200z(rc);
            hr = write_stream(outS, out_.p, produced - 1);     // every batch ends with the end marker: kept for the very end only
            if (hr != S_OK) return hr;
            processedIn += got; processedOut += produced - 1;
            if (progress) { hr = progress->SetRatioInfo(&processedIn, &processedOut); if (hr != S_OK) return hr; }
            if (got < batch) break;
        }
        const Byte endMark = 0;
        processedOut += 1;
        return write_stream(outS, &endMark, 1);
    }
};

class CLzma2Decoder final : public ICompressCoder, public ICompressSetDecoderProperties2, public ICompressSetFinishMode,
                            public ICompressGetInStreamProcessedSize, public ICompressSetCoderMt, public ICompressSetBufSize,
                            public ICompressSetMemLimit, public ICompressSetOutStreamSize, public ICompressSetInStream,
                            public ISequentialInStream, CoderBase {
    std::atomic<UInt32> refs_{0};
    Byte prop_ = 40; bool finishMode_ = false; UInt64 inProcessed_ = 0;
    static constexpr size_t kInStep = (size_t)256 << 20;         // granularity of reads / growth of the input staging
    static constexpr uint64_t kOutTarget = (uint64_t)1 << 30;    // decoded bytes per GPU batch
    static constexpr uint64_t kOutLimit = (uint64_t)48 << 30;    // a block that needs more staging than this is refused, never attempted
    PinnedBuf in_, out_;
    size_t inFill_ = 0; bool inEof_ = false;
    size_t batchSize_ = 0, batchPos_ = 0;                        // decoded batch in out_ the caller may take / has taken (pull mode)
    UInt64 produced_ = 0;                                        // decoded bytes of the whole stream (finish mode compares it with the unpack size)
    // pull mode (Lzma2Decoder.cpp:196-265): SetInStream + SetOutStreamSize, then Read() until it returns 0 bytes
    ISequentialInStream* pullIn_ = nullptr; bool pullDone_ = false;
    bool haveOutSize_ = false; UInt64 outSize_ = 0;
public:
    ~CLzma2Decoder() { if (pullIn_) pullIn_->Release(); }
    UInt64 processedIn = 0, processedOut = 0;
    HRESULT QueryInterface(const GUID& iid, void** out) override {
        *out = nullptr;
        if (iid == kIID_IUnknown || iid == b2z_iid(4, kIID_Coder)) *out = static_cast<ICompressCoder*>(this);
        else if (iid == b2z_iid(4, kIID_SetDecProps2)) *out = static_cast<ICompressSetDecoderProperties2*>(this);
        else if (iid == b2z_iid(4, kIID_SetFinishMode)) *out = static_cast<ICompressSetFinishMode*>(this);
        else if (iid == b2z_iid(4, kIID_GetInProcessed)) *out = static_cast<ICompressGetInStreamProcessedSize*>(this);
        else if (iid == b2z_iid(4, kIID_SetMt)) *out = static_cast<ICompressSetCoderMt*>(this);
        else if (iid == b2z_iid(4, kIID_SetBufSize)) *out = static_cast<ICompressSetBufSize*>(this);
        else if (iid == b2z_iid(4, kIID_SetMemLimit)) *out = static_cast<ICompressSetMemLimit*>(this);
        else if (iid == b2z_iid(4, kIID_SetOutStreamSize)) *out = static_cast<ICompressSetOutStreamSize*>(this);
        else if (iid == b2z_iid(4, kIID_SetInStream)) *out = static_cast<ICompressSetInStream*>(this);
        else if (iid == b2z_iid(3, kIID_SeqIn)) *out = static_cast<ISequentialInStream*>(this);
        else return E_NOINTERFACE;
        ++refs_; return S_OK;
    }
    UInt32 AddRef() override { return ++refs_; }
    UInt32 Release() override { UInt32 r = --refs_; if (!r) delete this; return r; }
    HRESULT SetInBufSize(UInt32, UInt32) override { return S_OK; }              // Lzma2Decoder.cpp:58-59: staging is sized by the stream here
    HRESULT SetOutBufSize(UInt32, UInt32) override { return S_OK; }
    HRESULT SetMemLimit(UInt64) override { return S_OK; }                       // limits the reference's MT block buffers; no equivalent
    HRESULT SetOutStreamSize(const UInt64* outSize) override {                  // Lzma2Decoder.cpp:208-243
        haveOutSize_ = outSize != nullptr; outSize_ = outSize ? *outSize : 0;
        pullDone_ = false; batchSize_ = batchPos_ = 0; processedIn = processedOut = 0; inProcessed_ = 0; produced_ = 0; inFill_ = 0; inEof_ = false;
        return S_OK;
    }
    HRESULT SetInStream(ISequentialInStream* in) override { if (in) in->AddRef(); if (pullIn_) pullIn_->Release(); pullIn_ = in; return S_OK; }
    HRESULT ReleaseInStream() override { if (pullIn_) pullIn_->Release(); pullIn_ = nullptr; return S_OK; }
    HRESULT Read(void* data, UInt32 size, UInt32* processed) override {
        if (processed) *processed = 0;
        if (!pullIn_) return E_FAIL;
        while (batchPos_ == batchSize_ && !pullDone_) {                         // current batch taken: decode the next one
            bool end = false;
            HRESULT hr = next_batch(pullIn_, &end);
            if (hr != S_OK) return hr;
            if (end) { pullDone_ = true; if (finishMode_ && haveOutSize_ && outSize_ != produced_ && batchSize_ == 0) return S_FALSE; }
        }
        size_t n = batchSize_ - batchPos_; if (n > size) n = size;
        memcpy(data, (const Byte*)out_.p + batchPos_, n); batchPos_ += n;
        if (processed) *processed = (UInt32)n;
        return S_OK;
    }
    HRESULT SetDecoderProperties2(const Byte* p, UInt32 size) override {       // Lzma2Decoder.cpp:40-48
        if (size != 1 || p[0] > 40) return E_NOTIMPL;
        prop_ = p[0]; return S_OK;
    }
    HRESULT SetFinishMode(UInt32 m) override { finishMode_ = m != 0; return S_OK; }
    HRESULT GetInStreamProcessedSize(UInt64* v) override { *v = inProcessed_; return S_OK; }
    HRESULT SetNumberOfThreads(UInt32) override { return S_OK; }                // parallelism = blocks in the stream

    // Decodes the next batch of whole dictionary-reset blocks into out_[0, batchSize_).  The packed stream is read piece by piece into
    // bounded pinned staging; a batch holds about kOutTarget decoded bytes (one block larger than that still goes alone, and a stream
    // with a single dictionary reset -- what the reference's encoders write for inputs below their block size -- is one block).
    // *end: the end marker has been consumed.  Output beyond the folder's unpack size is dropped (Lzma2Decoder.cpp:110-128).
    HRESULT next_batch(ISequentialInStream* inS, bool* end) {
        *end = false; batchSize_ = batchPos_ = 0;
        HRESULT hr = ensure_ctx(); if (hr != S_OK) return hr;
        for (;;) {
            if (!inEof_ && (in_.cap - inFill_ < kInStep / 2 + 1 || in_.cap == 0)) { if (!in_.reserve(inFill_ + kInStep + 1)) return E_OUTOFMEMORY; }   // + 1: room for an end marker
            if (!inEof_ && inFill_ + 1 < in_.cap) {
                size_t got = in_.cap - 1 - inFill_;
                hr = read_stream(inS, (Byte*)in_.p + inFill_, &got);
                if (hr != S_OK) return hr;
                if (got < in_.cap - 1 - inFill_) inEof_ = true;
                inFill_ += got;
            }
            size_t used = 0; uint64_t content = 0; uint32_t blocks = 0; int ended = 0;
            const int rc = b200z_lzma2_stream_prefix(in_.p, inFill_, kOutTarget, &used, &content, &blocks, &ended);
            if (rc) return S_FALSE;
            if (blocks == 0 && !ended) {
                if (inEof_) return S_FALSE;                              // the stream ends inside a block / has no end marker
                if (!in_.reserve(in_.cap + (in_.cap > kInStep ? in_.cap : kInStep))) return E_OUTOFMEMORY;
                continue;
            }
            if (content > kOutLimit) return E_OUTOFMEMORY;
            size_t produced = 0;
            if (blocks) {
                if (!out_.reserve((size_t)content + 64)) return E_OUTOFMEMORY;
                Byte* p = (Byte*)in_.p; size_t n = used; Byte saved = 0;
                if (!ended) { saved = p[used]; p[used] = 0; n = used + 1; }          // a batch cut out of a longer stream gets its own end marker
                const int drc = b200z_lzma2_decompress_host(ctx, p, n, prop_, out_.p, (size_t)content, &produced);
                if (!ended) p[used] = saved;
                if (drc) return hr_from_b200z(drc);
            }
            memmove(in_.p, (const Byte*)in_.p + used, inFill_ - used); inFill_ -= used;
            inProcessed_ += used; processedIn = inProcessed_; produced_ += produced;
            size_t give = produced;
            if (haveOutSize_) { const UInt64 left = outSize_ > processedOut ? outSize_ - processedOut : 0; if (give > left) give = (size_t)left; }
            batchSize_ = give; processedOut += give;
            if (ended) *end = true;
            return S_OK;
        }
    }

    HRESULT Code(ISequentialInStream* inS, ISequentialOutStream* outS, const UInt64*, const UInt64* outSize, ICompressProgressInfo* progress) override {
        SetOutStreamSize(outSize);
        for (;;) {
            bool end = false;
            HRESULT hr = next_batch(inS, &end);
            if (hr != S_OK) return hr;
            if (batchSize_) { hr = write_stream(outS, out_.p, batchSize_); if (hr != S_OK) return hr; }
            if (progress) { hr = progress->SetRatioInfo(&processedIn, &processedOut); if (hr != S_OK) return hr; }
            if (end) break;
        }
        if (finishMode_ && haveOutSize_ && outSize_ != produced_) return S_FALSE;      // Lzma2Decoder.cpp:177-183: the stream must end exactly there
        return S_OK;
    }
};

}  // namespace

ICompressCoder* b2z_new_lzma2_encoder(bool fast) { return new CLzma2Encoder(fast); }
ICompressCoder* b2z_new_lzma2_decoder() { return new CLzma2Decoder(); }
