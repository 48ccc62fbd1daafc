// emu_riscv.cpp -- TEST INFRASTRUCTURE ONLY: the RISC-V kernels of 7-zip-zstd_b200/csrc/b2z_filter.cu compiled for the host through
// tests/cuemu/cuemu.h (see there), with the launch shapes of b200z_filter_device.  tests/test_riscv_filter.py compiles it into a
// temporary library; never part of libb200z.so.
#define B2Z_CUEMU 1
#include "cuemu.h"
#include "../../7-zip-zstd_b200/csrc/b2z_filter.cu"

using namespace b2z;

extern "C" {

// RISC-V (method 0x0B) in place on `data`: map, scan and convert launches over a staged copy padded as b200z_filter_device pads it
void emu_riscv_filter(int enc, uint8_t* data, uint64_t n, uint32_t prop, uint32_t unitLog) {
    if (n < 8) return;
    const uint64_t nCta = ((n + B2Z_RV_CHUNK - 1) / B2Z_RV_CHUNK + B2Z_RV_THREADS - 1) / B2Z_RV_THREADS;
    std::vector<uint8_t> copy((size_t)nCta * B2Z_RV_SPAN + 64, 0xCD);
    memcpy(copy.data(), data, n);
    std::vector<uint8_t> maps((size_t)nCta * B2Z_RV_THREADS, 0xCD), ctaMaps(nCta, 0xCD), entry(nCta, 0xCD);
    cuemu::launch(dim3((uint32_t)nCta), dim3(B2Z_RV_THREADS), 0, [&] { riscv_map_kernel(copy.data(), n, unitLog, maps.data(), ctaMaps.data()); });
    cuemu::launch(dim3(1), dim3(1024), 0, [&] { riscv_scan_kernel(ctaMaps.data(), entry.data(), (uint32_t)nCta); });
    cuemu::launch(dim3((uint32_t)nCta), dim3(B2Z_RV_THREADS), 0, [&] { riscv_conv_kernel(copy.data(), data, n, prop, enc, unitLog, maps.data(), entry.data()); });
}

// the rule at one position (b2z_filter_ops.h): step | converts
uint32_t emu_riscv_scan(uint32_t w0, uint32_t w1) { return b2z_riscv_scan(w0, w1); }

}  // extern "C"
