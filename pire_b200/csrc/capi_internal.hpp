// capi_internal.hpp -- what the translation units behind include/pire_b200.h share: the scanner handle and a few
// helpers.  Not installed; the public surface is the C header.
#pragma once

#include "../../include/pire_b200.h"

#include <cuda_runtime.h>

#include <condition_variable>
#include <mutex>
#include <string>
#include <vector>

#include "dfa_tables.hpp"
#include "pire_image.hpp"
#include "scan_kernels.cuh"

namespace pire_b200 {

int Fail(int code, const std::string& what);
int FailCuda(cudaError_t err, const char* where);

#define CUDA_TRY(expr)                                   \
    do {                                                 \
        cudaError_t err__ = (expr);                      \
        if (err__ != cudaSuccess)                        \
            return ::pire_b200::FailCuda(err__, #expr);  \
    } while (0)

struct DeviceTables {
    uint8_t* hot8 = nullptr;
    uint8_t* noexit = nullptr;
    uint16_t* cls = nullptr;
    void* full = nullptr;
    DeviceFin* fin[2] = {nullptr, nullptr};
    uint32_t* priv_packed = nullptr;
    uint8_t* hot8_small = nullptr;
    uint8_t* flags = nullptr;
    uint32_t* acc_begin = nullptr;
    uint32_t* acc_ids = nullptr;
    uint64_t* weights = nullptr;
    uint32_t* accept_wide = nullptr;     // [states x accept_words], reference numbering: AcceptedRegexps as a bit set
    uint32_t* new_of_old = nullptr;      // [states]: reference numbering -> new (start states given by the caller)
    uint32_t* live = nullptr;            // ScanTables::live
    size_t full_bytes = 0;

    void Free();
};

struct HostWorkspace;                    // capi_host.cu: streams, pinned staging and device slots of one host-buffer call

} // namespace pire_b200

struct pire_gpu_scanner {
    pire_b200::Dfa dfa;
    pire_b200::ScanTables tab;
    pire_b200::DeviceTables dev;
    int device = -1;
    uint32_t variant = PIRE_GPU_VARIANT_AUTO;
    uint32_t auto_choice[2] = {0, 0};   // [uniform]: measured by pire_gpu_scanner_autoselect, 0 = heuristic
    uint32_t max_hot = pire_b200::kMaxHot;
    bool tuned = false;
    bool priv_ok = false;
    // counting kernel: 0 = automatic, 1 = accept lists, 2 = packed increments behind the look-ahead pass,
    // 3 = packed increments on every chunk (pire_gpu_scanner_set_count_mode; for tests and experiments)
    uint32_t count_mode = 0;
    double final_share = 0.0;       // share of a tune sample's steps that ended in a final state
    uint32_t accept_words = 1;      // 32-bit words per accept set: ceil(max(1, regexps) / 32)
    std::vector<uint32_t> hot_order;
    pire_b200::LaunchPlan plan[pire_b200::kVariantSlots][2];          // [variant][uniform]
    pire_b200::LaunchPlan plan_from[pire_b200::kVariantSlots][2];     // the same for per-string starts (no PRIV)

    // Workspaces of the host-buffer entry point: a call takes a free one (or makes one), so concurrent calls on one
    // handle do not serialise; the mutex guards this list only.
    std::mutex ws_mutex;
    std::vector<pire_b200::HostWorkspace*> ws_free;
};

namespace pire_b200 {

uint32_t ResolveVariant(const pire_gpu_scanner* sc, bool uniform = true);
// the variant a batch of n strings runs (pire_gpu_run_batch, pire_gpu_run_batch_ordered, pire_gpu_run_batch_from)
uint32_t BatchVariant(const pire_gpu_scanner* sc, bool uniform, uint64_t n);
bool IsUniform(const uint8_t* corpus, const uint64_t* offsets, uint64_t fixed_len);
void FillArgs(const pire_gpu_scanner* sc, ScanArgs* a, const uint8_t* corpus, const uint64_t* offsets, uint64_t fixed_len,
              uint64_t n, uint32_t flags);
int CheckRunnable(const pire_gpu_scanner* sc);
void FreeHostWorkspaces(pire_gpu_scanner* sc);          // capi_host.cu

} // namespace pire_b200
