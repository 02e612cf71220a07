// capi_slow.cu -- the Pire::SlowScanner entry points of include/pire_b200.h: a handle of its own (its state is a set
// of NFA states, not a StateIndex), the batch run, and the host-side Initialize / Next / Final on the parsed tables.
#include "capi_internal.hpp"

#include <cstring>
#include <new>

#include "slow_image.hpp"

struct pire_gpu_slow_scanner {
    pire_b200::Nfa nfa;
    int device = -1;
    uint32_t stride = 0;                // u32 words between two successor rows on the device
    uint64_t table_bytes = 0;
    uint64_t shared_bytes = 0;          // rows staged into shared memory per CTA (0: read through L1/L2)
    uint16_t* d_cls = nullptr;
    uint32_t* d_succ = nullptr;
    uint32_t* d_final = nullptr;
};

using namespace pire_b200;

namespace {

int UploadSlow(pire_gpu_slow_scanner* sc)
{
    const Nfa& f = sc->nfa;
    // rows padded to the kernel's stride: [letters][states][stride]
    std::vector<uint32_t> rows((size_t) f.letters * f.states * sc->stride, 0);
    for (size_t r = 0; r < (size_t) f.letters * f.states; ++r)
        std::memcpy(&rows[r * sc->stride], &f.succ[r * f.words], f.words * 4);
    CUDA_TRY(cudaSetDevice(sc->device));
    CUDA_TRY(cudaMalloc(&sc->d_cls, kMaxCharUnaligned * sizeof(uint16_t)));
    CUDA_TRY(cudaMalloc(&sc->d_succ, rows.size() * 4));
    CUDA_TRY(cudaMalloc(&sc->d_final, f.words * 4));
    CUDA_TRY(cudaMemcpy(sc->d_cls, f.class_of.data(), kMaxCharUnaligned * sizeof(uint16_t), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(sc->d_succ, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(sc->d_final, f.final_mask.data(), f.words * 4, cudaMemcpyHostToDevice));
    return PIRE_GPU_OK;
}

} // namespace

extern "C" {

int pire_gpu_slow_scanner_create(const void* image, size_t size, int device, pire_gpu_slow_scanner** out)
{
    if (!out)
        return Fail(PIRE_GPU_EINVAL, "out is null");
    *out = nullptr;
    pire_gpu_slow_scanner* sc = new (std::nothrow) pire_gpu_slow_scanner;
    if (!sc)
        return Fail(PIRE_GPU_EINVAL, "out of memory");
    std::string err;
    try {
        err = ParseSlowImage(image, size, &sc->nfa);
    } catch (const std::exception& e) {                 // bad_alloc on a huge (or lying) image
        err = std::string("slow scanner image: ") + e.what();
    }
    if (!err.empty()) {
        delete sc;
        return Fail(PIRE_GPU_EIMAGE, err);
    }
    if (sc->nfa.states > kSlowMaxStates) {
        const std::string what = "slow scanner with " + std::to_string(sc->nfa.states) + " states: at most "
                                 + std::to_string(kSlowMaxStates) + " are supported";
        delete sc;
        return Fail(PIRE_GPU_EUNSUPPORTED, what);
    }
    sc->stride = SlowRowStride(sc->nfa.states, sc->nfa.words);
    sc->table_bytes = (uint64_t) sc->nfa.letters * sc->nfa.states * sc->stride * 4;
    if (device >= 0) {
        int count = 0;
        cudaError_t ce = cudaGetDeviceCount(&count);
        if (ce != cudaSuccess || device >= count) {
            delete sc;
            return Fail(PIRE_GPU_ENODEVICE, ce != cudaSuccess ? std::string("no CUDA device: ") + cudaGetErrorString(ce)
                                                              : std::string("CUDA device index out of range"));
        }
        sc->device = device;
        sc->shared_bytes = SlowSharedBytes(sc->table_bytes, device);
        const int rc = UploadSlow(sc);
        if (rc != PIRE_GPU_OK) {
            pire_gpu_slow_scanner_destroy(sc);
            return rc;
        }
    }
    *out = sc;
    return PIRE_GPU_OK;
}

void pire_gpu_slow_scanner_destroy(pire_gpu_slow_scanner* sc)
{
    if (!sc)
        return;
    if (sc->device >= 0) {
        cudaSetDevice(sc->device);
        cudaFree(sc->d_cls);
        cudaFree(sc->d_succ);
        cudaFree(sc->d_final);
    }
    delete sc;
}

int pire_gpu_slow_scanner_info(const pire_gpu_slow_scanner* sc, pire_gpu_slow_info* out)
{
    if (!sc || !out)
        return Fail(PIRE_GPU_EINVAL, "null argument");
    std::memset(out, 0, sizeof(*out));
    out->states = sc->nfa.states;
    out->letters = sc->nfa.letters;
    out->regexps = sc->nfa.empty ? 0 : 1;
    out->set_words = sc->nfa.words;
    out->start = sc->nfa.start;
    out->empty = sc->nfa.empty ? 1 : 0;
    out->table_bytes = sc->table_bytes;
    out->shared_bytes = sc->shared_bytes;
    out->device = sc->device;
    return PIRE_GPU_OK;
}

int pire_gpu_slow_run_batch(const pire_gpu_slow_scanner* sc, const uint8_t* d_corpus, const uint64_t* d_offsets, uint64_t fixed_len,
                            uint64_t n, uint32_t flags, const uint32_t* d_start_sets, uint32_t* d_match_bits, uint32_t* d_sets,
                            void* stream)
{
    if (!sc)
        return Fail(PIRE_GPU_EINVAL, "null scanner");
    if (sc->device < 0)
        return Fail(PIRE_GPU_ENODEVICE, "host-only slow scanner handle (device -1)");
    if (flags & ~(PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END | PIRE_GPU_RUN_LINES))
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_slow_run_batch takes PIRE_GPU_RUN_BEGIN, PIRE_GPU_RUN_END and PIRE_GPU_RUN_LINES only");
    if ((flags & PIRE_GPU_RUN_LINES) && d_start_sets)
        return Fail(PIRE_GPU_EINVAL, "PIRE_GPU_RUN_LINES walks every line from Initialize(): no start sets");
    if ((flags & PIRE_GPU_RUN_LINES) && !d_offsets)
        return Fail(PIRE_GPU_EINVAL, "PIRE_GPU_RUN_LINES needs the line offsets");
    if (n == 0)
        return PIRE_GPU_OK;
    if (!d_corpus && (d_offsets || fixed_len != 0))
        return Fail(PIRE_GPU_EINVAL, "null corpus with non-empty strings");
    if (n > (1ull << 40))
        return Fail(PIRE_GPU_EINVAL, "too many strings");
    CUDA_TRY(cudaSetDevice(sc->device));
    SlowArgs a;
    std::memset(&a, 0, sizeof(a));
    a.corpus = d_corpus;
    a.offsets = d_offsets;
    a.trim = (flags & PIRE_GPU_RUN_LINES) ? 1 : 0;
    a.fixed_len = d_offsets ? 0 : fixed_len;
    a.n = n;
    a.cls = sc->d_cls;
    a.succ = sc->d_succ;
    a.final_mask = sc->d_final;
    a.states = sc->nfa.states;
    a.words = sc->nfa.words;
    a.start = sc->nfa.start;
    a.with_begin = (flags & PIRE_GPU_RUN_BEGIN) ? 1 : 0;
    a.with_end = (flags & PIRE_GPU_RUN_END) ? 1 : 0;
    a.shared_rows = (uint32_t) sc->shared_bytes;
    a.start_sets = d_start_sets;
    a.match_bits = d_match_bits;
    a.sets = d_sets;
    CUDA_TRY(LaunchSlow(a, sc->device, static_cast<cudaStream_t>(stream)));
    return PIRE_GPU_OK;
}

int pire_gpu_slow_initial(const pire_gpu_slow_scanner* sc, uint32_t* set)
{
    if (!sc || !set)
        return Fail(PIRE_GPU_EINVAL, "null argument");
    std::memset(set, 0, sc->nfa.words * 4);
    set[sc->nfa.start / 32] = 1u << (sc->nfa.start % 32);
    return PIRE_GPU_OK;
}

int pire_gpu_slow_next(const pire_gpu_slow_scanner* sc, const uint32_t* set, uint32_t ch, uint32_t* out)
{
    if (!sc || !set || !out)
        return Fail(PIRE_GPU_EINVAL, "null argument");
    if (ch >= kMaxCharUnaligned)
        return Fail(PIRE_GPU_EINVAL, "symbol past EndMark");
    sc->nfa.Next(set, ch, out);
    return PIRE_GPU_OK;
}

int pire_gpu_slow_final(const pire_gpu_slow_scanner* sc, const uint32_t* set)
{
    if (!sc || !set)
        return Fail(PIRE_GPU_EINVAL, "null argument");
    return sc->nfa.Final(set) ? 1 : 0;
}

} // extern "C"
