// capi.cu -- the extern "C" boundary declared in include/pire_b200.h.
//
// Host side of the scan path: ingest the reference's Scanner::Save() stream
// (pire_image.cpp), build and upload the device tables (dfa_tables.cpp), launch
// the sm_90a kernels (scan_kernels.cu).  There is deliberately no CPU scan
// here: without a CUDA device every run entry point fails with
// PIRE_GPU_ENODEVICE.
#include "capi_internal.hpp"

#include <cstdlib>
#include <cstring>
#include <exception>
#include <new>

#include "synth.h"

using namespace pire_b200;

namespace pire_b200 {

namespace {
thread_local std::string g_error;
}

int Fail(int code, const std::string& what)
{
    g_error = what;
    return code;
}

int FailCuda(cudaError_t err, const char* where)
{
    g_error = std::string(where) + ": " + cudaGetErrorString(err);
    return PIRE_GPU_ECUDA;
}

void DeviceTables::Free()
{
    cudaFree(hot8);
    cudaFree(noexit);
    cudaFree(cls);
    cudaFree(full);
    cudaFree(fin[0]);
    cudaFree(fin[1]);
    cudaFree(priv_packed);
    cudaFree(hot8_small);
    cudaFree(flags);
    cudaFree(acc_begin);
    cudaFree(acc_ids);
    cudaFree(weights);
    cudaFree(accept_wide);
    cudaFree(new_of_old);
    cudaFree(live);
    *this = DeviceTables();
}

uint32_t ResolveVariant(const pire_gpu_scanner* sc, bool uniform)
{
    if (sc->variant >= PIRE_GPU_VARIANT_PLAIN && sc->variant <= PIRE_GPU_VARIANT_LOOK_RING1) {
        if (sc->variant >= PIRE_GPU_VARIANT_LOOK && !sc->tab.look_ok)
            return PIRE_GPU_VARIANT_PRED;       // an exit of the resting state is cold: no look-ahead set
        return sc->variant;
    }
    if (sc->auto_choice[uniform ? 1 : 0])
        return sc->auto_choice[uniform ? 1 : 0];
    // AUTO: predication pays when lanes outside the resident state would
    // collide with it in the banks, i.e. for large (glued) automata -- in the uniform kernel, which is bound
    // by shared-memory wavefronts.  The CSR kernels (generic, lines) are bound by instruction issue on short
    // strings, where the filter's two extra instructions per byte cost more than the conflicts they save.
    if (!uniform)
        return PIRE_GPU_VARIANT_PLAIN;
    // the look-ahead filter (5.5 instructions per byte, two strings per lane) is chosen over the exit filter for the
    // glued benchmark scanner; it needs the look-ahead set (every exit of the resting state hot)
    if (sc->tab.states > 64)
        return sc->tab.look_ok ? PIRE_GPU_VARIANT_LOOK : PIRE_GPU_VARIANT_PRED;
    return PIRE_GPU_VARIANT_PLAIN;
}

uint32_t BatchVariant(const pire_gpu_scanner* sc, bool uniform, uint64_t n)
{
    uint32_t variant = ResolveVariant(sc, uniform);
    if (variant == PIRE_GPU_VARIANT_PRIV && !(uniform && sc->priv_ok))
        variant = PIRE_GPU_VARIANT_PLAIN;       // the private-row kernel exists for uniform batches only
    if (variant == PIRE_GPU_VARIANT_LOOK && uniform && sc->variant == PIRE_GPU_VARIANT_AUTO) {
        // two strings per lane pay when every resident warp gets a pair of units; a smaller batch (a 64 MiB chunk of
        // the host entry point, say) keeps more warps busy with one string per lane
        const LaunchPlan& two = sc->plan[PIRE_GPU_VARIANT_LOOK][1];
        const uint64_t pairs = ((n + 31) / 32 + 1) / 2;
        if (pairs < (uint64_t) two.grid * (uint64_t) (two.block / 32))
            variant = PIRE_GPU_VARIANT_LOOK1;
    }
    return variant;
}

namespace {

int Upload(pire_gpu_scanner* sc)
{
    if (sc->device < 0)
        return PIRE_GPU_OK;
    CUDA_TRY(cudaSetDevice(sc->device));
    sc->dev.Free();
    const ScanTables& t = sc->tab;
    DeviceTables& d = sc->dev;
    CUDA_TRY(cudaMalloc(&d.hot8, t.hot8.size()));
    CUDA_TRY(cudaMemcpy(d.hot8, t.hot8.data(), t.hot8.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMalloc(&d.noexit, t.noexit.size()));
    CUDA_TRY(cudaMemcpy(d.noexit, t.noexit.data(), t.noexit.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMalloc(&d.cls, 512));
    CUDA_TRY(cudaMemcpy(d.cls, t.cls.data(), 512, cudaMemcpyHostToDevice));
    const void* full_src = t.wide ? (const void*) t.full32.data() : (const void*) t.full16.data();
    d.full_bytes = t.wide ? t.full32.size() * 4 : t.full16.size() * 2;
    CUDA_TRY(cudaMalloc(&d.full, d.full_bytes));
    CUDA_TRY(cudaMemcpy(d.full, full_src, d.full_bytes, cudaMemcpyHostToDevice));
    for (int w = 0; w < 2; ++w) {
        static_assert(sizeof(FinEntry) == sizeof(DeviceFin), "fin layout");
        size_t bytes = t.fin[w].size() * sizeof(FinEntry);
        CUDA_TRY(cudaMalloc(&d.fin[w], bytes));
        CUDA_TRY(cudaMemcpy(d.fin[w], t.fin[w].data(), bytes, cudaMemcpyHostToDevice));
    }
    CUDA_TRY(cudaMalloc(&d.priv_packed, t.priv_packed.size() * 4));
    CUDA_TRY(cudaMemcpy(d.priv_packed, t.priv_packed.data(), t.priv_packed.size() * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMalloc(&d.hot8_small, t.hot8_small.size()));
    CUDA_TRY(cudaMemcpy(d.hot8_small, t.hot8_small.data(), t.hot8_small.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMalloc(&d.flags, t.flags_new.size()));
    CUDA_TRY(cudaMemcpy(d.flags, t.flags_new.data(), t.flags_new.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMalloc(&d.acc_begin, t.acc_begin_new.size() * 4));
    CUDA_TRY(cudaMemcpy(d.acc_begin, t.acc_begin_new.data(), t.acc_begin_new.size() * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMalloc(&d.acc_ids, t.acc_ids_new.size() * 4 + 4));
    if (!t.acc_ids_new.empty())
        CUDA_TRY(cudaMemcpy(d.acc_ids, t.acc_ids_new.data(), t.acc_ids_new.size() * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMalloc(&d.weights, t.weights.size() * 8 + 8));
    if (!t.weights.empty())
        CUDA_TRY(cudaMemcpy(d.weights, t.weights.data(), t.weights.size() * 8, cudaMemcpyHostToDevice));
    // AcceptedRegexps as a bit set per state (reference numbering), for automata with more than 32 regexps:
    // pire_gpu_accept_sets gathers rows of this table by StateIndex
    {
        const uint32_t regs = sc->dfa.regexps ? sc->dfa.regexps : 1;
        sc->accept_words = (regs + 31) / 32;
        std::vector<uint32_t> wide((size_t) sc->dfa.states * sc->accept_words, 0);
        for (uint32_t st = 0; st < sc->dfa.states; ++st)
            for (uint32_t k = sc->dfa.acc_begin[st]; k < sc->dfa.acc_begin[st + 1]; ++k) {
                const uint32_t id = sc->dfa.acc_ids[k];
                if (id < regs)
                    wide[(size_t) st * sc->accept_words + id / 32] |= 1u << (id % 32);
            }
        CUDA_TRY(cudaMalloc(&d.accept_wide, wide.size() * 4));
        CUDA_TRY(cudaMemcpy(d.accept_wide, wide.data(), wide.size() * 4, cudaMemcpyHostToDevice));
    }
    CUDA_TRY(cudaMalloc(&d.live, t.live.size() * 4 + 4));
    if (!t.live.empty())
        CUDA_TRY(cudaMemcpy(d.live, t.live.data(), t.live.size() * 4, cudaMemcpyHostToDevice));
    // tuning renumbers the states: the map is rebuilt with the other tables
    CUDA_TRY(cudaMalloc(&d.new_of_old, t.new_of_old.size() * 4 + 4));
    if (!t.new_of_old.empty())
        CUDA_TRY(cudaMemcpy(d.new_of_old, t.new_of_old.data(), t.new_of_old.size() * 4, cudaMemcpyHostToDevice));
    sc->priv_ok = false;
    for (int v = kVariantPlain; v <= kVariantLookRing1; ++v)
        for (int u = 0; u < 2; ++u) {
            cudaError_t pe = PlanScan(sc->device, t.hot, t.hot_small, t.priv_rows, v, u != 0, &sc->plan[v][u]);
            if (v == kVariantPriv && u == 1) {
                sc->priv_ok = pe == cudaSuccess;     // needs ~225 KB of shared memory per CTA
                if (pe != cudaSuccess)
                    (void) cudaGetLastError();
                continue;
            }
            if (pe != cudaSuccess)
                return FailCuda(pe, "PlanScan");
            if (v != kVariantPriv)
                CUDA_TRY(PlanScan(sc->device, t.hot, t.hot_small, t.priv_rows, v, u != 0, &sc->plan_from[v][u], true));
        }
    return PIRE_GPU_OK;
}

void Rebuild(pire_gpu_scanner* sc)
{
    BuildScanTables(sc->dfa, sc->hot_order, sc->max_hot, &sc->tab);
}

} // namespace

bool IsUniform(const uint8_t* corpus, const uint64_t* offsets, uint64_t fixed_len)
{
    return offsets == nullptr && fixed_len != 0 && fixed_len % 32 == 0 && fixed_len <= 0xffffffe0ull
           && (reinterpret_cast<uintptr_t>(corpus) & 31) == 0;
}

void FillArgs(const pire_gpu_scanner* sc, ScanArgs* a, const uint8_t* corpus, const uint64_t* offsets,
              uint64_t fixed_len, uint64_t n, uint32_t flags)
{
    const ScanTables& t = sc->tab;
    std::memset(a, 0, sizeof(*a));
    a->corpus = corpus;
    a->offsets = offsets;
    a->fixed_len = fixed_len;
    a->n = n;
    a->hot8 = sc->dev.hot8;
    a->noexit = sc->dev.noexit;
    a->cls = sc->dev.cls;
    a->full = sc->dev.full;
    a->fin = sc->dev.fin[(flags & PIRE_GPU_RUN_END) ? 1 : 0];
    a->hot = t.hot;
    a->letters = t.letters;
    a->wide = t.wide ? 1 : 0;
    a->start = t.start[(flags & PIRE_GPU_RUN_BEGIN) ? 1 : 0];
    a->trim = (offsets && (flags & PIRE_GPU_RUN_LINES)) ? 1 : 0;
    a->exit_bitmap0 = t.exit_bitmap0;
    a->look_bitmap = t.look_bitmap;
    a->look_bitmap64 = t.look_bitmap64;
    a->priv_packed = sc->dev.priv_packed;
    a->priv_rows = t.priv_rows;
    a->hot8_small = sc->dev.hot8_small;
    a->hot_small = t.hot_small;
}

int CheckRunnable(const pire_gpu_scanner* sc)
{
    if (!sc)
        return Fail(PIRE_GPU_EINVAL, "null scanner handle");
    if (sc->device < 0)
        return Fail(PIRE_GPU_ENODEVICE, "host-only scanner handle: the scan path has no CPU fallback");
    return PIRE_GPU_OK;
}

} // namespace pire_b200

extern "C" {

int pire_gpu_scanner_create(const void* image, size_t size, int device, pire_gpu_scanner** out)
{
    if (!out)
        return Fail(PIRE_GPU_EINVAL, "out is null");
    *out = nullptr;
    pire_gpu_scanner* sc = new (std::nothrow) pire_gpu_scanner;
    if (!sc)
        return Fail(PIRE_GPU_EINVAL, "out of memory");
    std::string err;
    try {
        err = ParsePireImage(image, size, &sc->dfa);
    } catch (const std::exception& e) {                 // bad_alloc / length_error on a huge (or lying) image
        err = std::string("scanner image: ") + e.what();
    }
    if (!err.empty()) {
        delete sc;
        return Fail(PIRE_GPU_EIMAGE, err);
    }
    sc->device = -1;
    if (device >= 0) {
        int count = 0;
        cudaError_t ce = cudaGetDeviceCount(&count);
        if (ce != cudaSuccess || device >= count) {
            delete sc;
            return Fail(PIRE_GPU_ENODEVICE, ce != cudaSuccess ? std::string("no CUDA device: ") + cudaGetErrorString(ce)
                                                              : std::string("CUDA device index out of range"));
        }
        ce = PrepareScanKernels(device);
        if (ce != cudaSuccess) {
            delete sc;
            return FailCuda(ce, "PrepareScanKernels");
        }
        sc->device = device;
    }
    try {
        sc->hot_order = StaticHotOrder(sc->dfa);
        Rebuild(sc);
    } catch (const std::exception& e) {
        delete sc;
        return Fail(PIRE_GPU_EIMAGE, std::string("building the scan tables: ") + e.what());
    }
    int rc = Upload(sc);
    if (rc != PIRE_GPU_OK) {
        pire_gpu_scanner_destroy(sc);
        return rc;
    }
    *out = sc;
    return PIRE_GPU_OK;
}

void pire_gpu_scanner_destroy(pire_gpu_scanner* sc)
{
    if (!sc)
        return;
    if (sc->device >= 0) {
        cudaSetDevice(sc->device);
        sc->dev.Free();
        FreeHostWorkspaces(sc);
    }
    delete sc;
}

int pire_gpu_scanner_info(const pire_gpu_scanner* sc, pire_gpu_info* out)
{
    if (!sc || !out)
        return Fail(PIRE_GPU_EINVAL, "null argument");
    std::memset(out, 0, sizeof(*out));
    out->states = sc->dfa.states;
    out->letters = sc->dfa.letters;
    out->regexps = sc->dfa.regexps;
    out->initial = sc->dfa.initial;
    out->empty = sc->dfa.empty ? 1 : 0;
    out->hot_rows = sc->tab.hot;
    out->variant = ResolveVariant(sc);
    out->tuned = sc->tuned ? 1 : 0;
    out->table_bytes = sc->tab.wide ? sc->tab.full32.size() * 4 : sc->tab.full16.size() * 2;
    out->shared_bytes = ResolveVariant(sc) == PIRE_GPU_VARIANT_PRIV ? ScanSharedBytes(sc->tab.hot_small, sc->tab.priv_rows)
                                                                    : ScanSharedBytes(sc->tab.hot, 0);
    out->device = sc->device;
    return PIRE_GPU_OK;
}

int pire_gpu_scanner_set_variant(pire_gpu_scanner* sc, uint32_t variant)
{
    if (!sc || variant > PIRE_GPU_VARIANT_LOOK_RING1)
        return Fail(PIRE_GPU_EINVAL, "bad variant");
    sc->variant = variant;
    return PIRE_GPU_OK;
}

int pire_gpu_scanner_set_max_hot(pire_gpu_scanner* sc, uint32_t max_hot_rows)
{
    if (!sc || max_hot_rows == 0)
        return Fail(PIRE_GPU_EINVAL, "bad max_hot_rows");
    sc->max_hot = max_hot_rows < kMaxHot ? max_hot_rows : kMaxHot;
    try {
        Rebuild(sc);
    } catch (const std::exception& e) {
        return Fail(PIRE_GPU_EINVAL, std::string("building the scan tables: ") + e.what());
    }
    return Upload(sc);
}

int pire_gpu_scanner_set_count_mode(pire_gpu_scanner* sc, uint32_t mode)
{
    if (!sc || mode > PIRE_GPU_COUNT_EVERY_CHUNK)
        return Fail(PIRE_GPU_EINVAL, "bad count mode");
    sc->count_mode = mode;
    return PIRE_GPU_OK;
}

// Per-string starts (pire_gpu_run_batch_from): n words of StateIndex, mapped and stepped through BeginMark in the kernels.
static void SetStarts(const pire_gpu_scanner* sc, ScanArgs* a, const uint32_t* d_start, uint32_t flags)
{
    a->starts = d_start;
    a->new_of_old = sc->dev.new_of_old;
    a->states = sc->tab.states;
    a->with_begin = (flags & PIRE_GPU_RUN_BEGIN) ? 1 : 0;
    a->begin_class = sc->tab.begin_class;
}

// pire_gpu_run_batch once its arguments are checked; d_start = per-string starts or null
static int RunBatch(const pire_gpu_scanner* sc, const uint8_t* d_corpus, const uint64_t* d_offsets, uint64_t fixed_len, uint64_t n,
                    uint32_t flags, const uint32_t* d_start, uint32_t* d_match_bits, uint32_t* d_accept_masks, uint32_t* d_state_idx,
                    void* stream)
{
    if (n > (1ull << 40))
        return Fail(PIRE_GPU_EINVAL, "too many strings");
    CUDA_TRY(cudaSetDevice(sc->device));
    ScanArgs a;
    FillArgs(sc, &a, d_corpus, d_offsets, fixed_len, n, flags);
    a.match_bits = d_match_bits;
    a.accept_masks = d_accept_masks;
    a.state_idx = d_state_idx;
    const bool uniform = IsUniform(d_corpus, d_offsets, fixed_len);
    uint32_t variant = BatchVariant(sc, uniform, n);
    const LaunchPlan* plan = &sc->plan[variant][uniform ? 1 : 0];
    if (d_start) {
        SetStarts(sc, &a, d_start, flags);
        if (variant == PIRE_GPU_VARIANT_PRIV)
            variant = PIRE_GPU_VARIANT_PLAIN;       // no private-row kernel with starts: PLAIN's walk
        plan = &sc->plan_from[variant][uniform ? 1 : 0];
    }
    CUDA_TRY(LaunchScan(a, (int) variant, uniform, *plan, static_cast<cudaStream_t>(stream)));
    return PIRE_GPU_OK;
}

int pire_gpu_run_batch(const pire_gpu_scanner* sc, const uint8_t* d_corpus, const uint64_t* d_offsets,
                       uint64_t fixed_len, uint64_t n, uint32_t flags,
                       uint32_t* d_match_bits, uint32_t* d_accept_masks, uint32_t* d_state_idx, void* stream)
{
    int rc = CheckRunnable(sc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (flags & ~(PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END | PIRE_GPU_RUN_LINES))
        return Fail(PIRE_GPU_EINVAL, "unknown run flags");
    if (n == 0)
        return PIRE_GPU_OK;
    if (!d_corpus && (d_offsets || fixed_len != 0))
        return Fail(PIRE_GPU_EINVAL, "null corpus with non-empty strings");
    return RunBatch(sc, d_corpus, d_offsets, fixed_len, n, flags, nullptr, d_match_bits, d_accept_masks, d_state_idx, stream);
}

static int PrefixOrSuffix(const pire_gpu_scanner* sc, const uint8_t* d_corpus, const uint64_t* d_offsets, uint64_t fixed_len,
                          uint64_t n, uint32_t flags, int shortest, bool reverse, uint32_t* d_len, void* stream)
{
    int rc = CheckRunnable(sc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (flags & ~(PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END | PIRE_GPU_RUN_LINES))
        return Fail(PIRE_GPU_EINVAL, "unknown run flags");
    if (n == 0)
        return PIRE_GPU_OK;
    if (!d_len || (!d_corpus && (d_offsets || fixed_len != 0)))
        return Fail(PIRE_GPU_EINVAL, "null corpus or output");
    if (!d_offsets && fixed_len > 0xfffffffeull)
        return Fail(PIRE_GPU_EINVAL, "strings longer than 4 GiB");
    CUDA_TRY(cudaSetDevice(sc->device));
    ScanArgs a;
    FillArgs(sc, &a, d_corpus, d_offsets, fixed_len, n, flags);
    a.flags = sc->dev.flags;
    a.initial = sc->tab.initial;
    // the mark stepped before the bytes and the one stepped after them: Begin..End for a prefix scan
    // (run.h:282-283,:286-290), End..Begin for a suffix scan (run.h:321-322,:336-340)
    const uint32_t begin = (flags & PIRE_GPU_RUN_BEGIN) ? 1 : 0, end = (flags & PIRE_GPU_RUN_END) ? 1 : 0;
    a.with_begin = reverse ? end : begin;
    a.begin_class = reverse ? sc->tab.end_class : sc->tab.begin_class;
    a.through_end = reverse ? begin : end;
    a.end_class = reverse ? sc->tab.begin_class : sc->tab.end_class;
    a.prefix_len = d_len;
    a.first_final_hot = sc->tab.first_final_hot;
    a.uniform = (!reverse && IsUniform(d_corpus, d_offsets, fixed_len)) ? 1 : 0;
    CUDA_TRY(LaunchPrefix(a, shortest != 0, reverse, sc->device, static_cast<cudaStream_t>(stream)));
    return PIRE_GPU_OK;
}

int pire_gpu_prefix_batch(const pire_gpu_scanner* sc, const uint8_t* d_corpus, const uint64_t* d_offsets,
                          uint64_t fixed_len, uint64_t n, uint32_t flags, int shortest, uint32_t* d_prefix_len, void* stream)
{
    return PrefixOrSuffix(sc, d_corpus, d_offsets, fixed_len, n, flags, shortest, false, d_prefix_len, stream);
}

int pire_gpu_suffix_batch(const pire_gpu_scanner* sc, const uint8_t* d_corpus, const uint64_t* d_offsets,
                          uint64_t fixed_len, uint64_t n, uint32_t flags, int shortest, uint32_t* d_suffix_len, void* stream)
{
    return PrefixOrSuffix(sc, d_corpus, d_offsets, fixed_len, n, flags, shortest, true, d_suffix_len, stream);
}

// The counting fields of every count entry point (HalfFinalScanner::TakeAction), count mode included.
static void SetCounting(const pire_gpu_scanner* sc, ScanArgs* a, uint32_t flags)
{
    a->flags = sc->dev.flags;
    a->end_class = sc->tab.end_class;
    a->through_end = (flags & PIRE_GPU_RUN_END) ? 1 : 0;
    a->acc_begin = sc->dev.acc_begin;
    a->acc_ids = sc->dev.acc_ids;
    a->first_final_hot = sc->tab.first_final_hot;
    a->begin_class = sc->tab.begin_class;
    a->initial = sc->tab.initial;
    a->with_begin = (flags & PIRE_GPU_RUN_BEGIN) ? 1 : 0;
    a->regexps = sc->dfa.regexps ? sc->dfa.regexps : 1;
    a->weights = sc->dev.weights;
    a->count_words = sc->count_mode == 1 ? 0 : sc->tab.count_words;
    a->count_always = (sc->count_mode == 3 || (sc->count_mode == 0 && sc->final_share > 0.025)) ? 1 : 0;
}

int pire_gpu_count_batch(const pire_gpu_scanner* sc, const uint8_t* d_corpus, const uint64_t* d_offsets,
                         uint64_t fixed_len, uint64_t n, uint32_t flags, uint32_t* d_counts, uint32_t* d_match_bits,
                         void* stream)
{
    int rc = CheckRunnable(sc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (flags & ~(PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END | PIRE_GPU_RUN_LINES))
        return Fail(PIRE_GPU_EINVAL, "unknown run flags");
    if (n == 0)
        return PIRE_GPU_OK;
    if (!d_counts || (!d_corpus && (d_offsets || fixed_len != 0)))
        return Fail(PIRE_GPU_EINVAL, "null corpus or output");
    CUDA_TRY(cudaSetDevice(sc->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ScanArgs a;
    FillArgs(sc, &a, d_corpus, d_offsets, fixed_len, n, flags);
    SetCounting(sc, &a, flags);
    a.counts = d_counts;
    a.match_bits = d_match_bits;
    a.uniform = IsUniform(d_corpus, d_offsets, fixed_len) ? 1 : 0;
    CUDA_TRY(cudaMemsetAsync(d_counts, 0, (size_t) n * a.regexps * 4, st));
    CUDA_TRY(LaunchCount(a, sc->device, st));
    return PIRE_GPU_OK;
}

int pire_gpu_count_batch_from(const pire_gpu_scanner* sc, const uint8_t* d_corpus, const uint64_t* d_offsets,
                              uint64_t fixed_len, uint64_t n, uint32_t flags, const uint32_t* d_start, uint64_t* d_counts,
                              uint32_t* d_match_bits, uint32_t* d_state_idx, void* stream)
{
    int rc = CheckRunnable(sc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (flags & ~(PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END))
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_count_batch_from takes PIRE_GPU_RUN_BEGIN and PIRE_GPU_RUN_END only");
    if (n == 0)
        return PIRE_GPU_OK;
    if (!d_counts)
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_count_batch_from needs n rows of max(1, regexps) u64 counters");
    if (!d_corpus && (d_offsets || fixed_len != 0))
        return Fail(PIRE_GPU_EINVAL, "null corpus with non-empty strings");
    if (n > (1ull << 40))
        return Fail(PIRE_GPU_EINVAL, "too many strings");
    CUDA_TRY(cudaSetDevice(sc->device));
    ScanArgs a;
    FillArgs(sc, &a, d_corpus, d_offsets, fixed_len, n, flags);
    SetCounting(sc, &a, flags);
    if (d_start)
        SetStarts(sc, &a, d_start, flags);
    a.counts64 = reinterpret_cast<unsigned long long*>(d_counts);
    a.match_bits = d_match_bits;
    a.state_idx = d_state_idx;
    a.uniform = IsUniform(d_corpus, d_offsets, fixed_len) ? 1 : 0;
    CUDA_TRY(LaunchCount(a, sc->device, static_cast<cudaStream_t>(stream), true));
    return PIRE_GPU_OK;
}

int pire_gpu_match_ends_batch_from(const pire_gpu_scanner* sc, const uint8_t* d_corpus, const uint64_t* d_offsets,
                                   uint64_t fixed_len, uint64_t n, uint32_t flags, const uint32_t* d_start, uint64_t* d_pos,
                                   uint32_t* d_strings, uint64_t* d_ends, uint32_t* d_ids, uint64_t capacity, uint64_t* d_found,
                                   uint32_t* d_match_bits, uint32_t* d_state_idx, void* stream)
{
    int rc = CheckRunnable(sc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (flags & ~(PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END))
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_match_ends_batch_from takes PIRE_GPU_RUN_BEGIN and PIRE_GPU_RUN_END only");
    if (n == 0)
        return PIRE_GPU_OK;
    if (!d_found)
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_match_ends_batch_from needs a device word for the number of entries");
    if (!d_corpus && (d_offsets || fixed_len != 0))
        return Fail(PIRE_GPU_EINVAL, "null corpus with non-empty strings");
    if (n >= (1ull << 32))
        return Fail(PIRE_GPU_EINVAL, "too many strings: string indices are u32");
    CUDA_TRY(cudaSetDevice(sc->device));
    ScanArgs a;
    FillArgs(sc, &a, d_corpus, d_offsets, fixed_len, n, flags);
    SetCounting(sc, &a, flags);
    if (d_start)
        SetStarts(sc, &a, d_start, flags);
    a.match_bits = d_match_bits;
    a.state_idx = d_state_idx;
    a.uniform = IsUniform(d_corpus, d_offsets, fixed_len) ? 1 : 0;
    a.pos = d_pos;
    a.strings = d_strings;
    a.ends = d_ends;
    a.ids = d_ids;
    a.ends_capacity = capacity;
    a.found = reinterpret_cast<unsigned long long*>(d_found);
    CUDA_TRY(LaunchMatchEndsBatch(a, sc->device, static_cast<cudaStream_t>(stream)));
    return PIRE_GPU_OK;
}

int pire_gpu_match_ends_lines(const pire_gpu_scanner* sc, const uint8_t* d_text, const uint64_t* d_line_offsets,
                              uint64_t n_lines, uint32_t flags, uint32_t* d_lines, uint64_t* d_ends, uint32_t* d_ids,
                              uint64_t capacity, uint64_t* d_found, uint32_t* d_match_bits, uint32_t* d_state_idx, void* stream)
{
    int rc = CheckRunnable(sc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (flags & ~(PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END | PIRE_GPU_RUN_LINES))
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_match_ends_lines takes PIRE_GPU_RUN_BEGIN, PIRE_GPU_RUN_END and PIRE_GPU_RUN_LINES only");
    if (!d_found)
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_match_ends_lines needs a device word for the number of entries");
    if (!d_line_offsets)
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_match_ends_lines needs the line offsets");
    if (n_lines == 0)
        return PIRE_GPU_OK;
    if (!d_text)
        return Fail(PIRE_GPU_EINVAL, "null text with lines");
    if (n_lines >= (1ull << 32))
        return Fail(PIRE_GPU_EINVAL, "too many lines: line indices are u32");
    CUDA_TRY(cudaSetDevice(sc->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ScanArgs a;
    FillArgs(sc, &a, d_text, d_line_offsets, 0, n_lines, flags | PIRE_GPU_RUN_LINES);
    SetCounting(sc, &a, flags);
    a.match_bits = d_match_bits;
    a.state_idx = d_state_idx;
    a.strings = d_lines;
    a.ends = d_ends;
    a.ids = d_ids;
    a.ends_capacity = capacity;
    a.found = reinterpret_cast<unsigned long long*>(d_found);
    if (d_match_bits)
        CUDA_TRY(cudaMemsetAsync(d_match_bits, 0, (size_t) ((n_lines + 31) / 32) * 4, st));
    CUDA_TRY(LaunchMatchEndsLines(a, sc->device, st));
    return PIRE_GPU_OK;
}

uint32_t pire_gpu_accept_words(const pire_gpu_scanner* sc) { return sc ? sc->accept_words : 0; }

int pire_gpu_accept_sets(const pire_gpu_scanner* sc, const uint32_t* d_state_idx, uint64_t n, uint32_t* d_accept_sets, void* stream)
{
    int rc = CheckRunnable(sc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (n == 0)
        return PIRE_GPU_OK;
    if (!d_state_idx || !d_accept_sets)
        return Fail(PIRE_GPU_EINVAL, "null state indices or output");
    CUDA_TRY(cudaSetDevice(sc->device));
    CUDA_TRY(LaunchAcceptGather(sc->dev.accept_wide, sc->dfa.states, sc->accept_words, d_state_idx, n, d_accept_sets,
                                static_cast<cudaStream_t>(stream)));
    return PIRE_GPU_OK;
}

int pire_gpu_length_order(const uint64_t* d_offsets, uint64_t n, uint32_t* d_order, int device, void* stream)
{
    if (n && (!d_offsets || !d_order))
        return Fail(PIRE_GPU_EINVAL, "null offsets or order");
    if (n >= (1ull << 31))
        return Fail(PIRE_GPU_EINVAL, "too many strings for a length order");
    CUDA_TRY(cudaSetDevice(device));
    CUDA_TRY(LengthOrder(d_offsets, n, d_order, static_cast<cudaStream_t>(stream)));
    return PIRE_GPU_OK;
}

static int RunCsr(const pire_gpu_scanner* sc, const uint8_t* d_corpus, const uint64_t* d_offsets, const uint32_t* d_order,
                  uint64_t n, uint32_t flags, uint32_t* d_match_bits, uint32_t* d_accept_masks, uint32_t* d_state_idx,
                  void* stream, const uint32_t* d_start = nullptr);

int pire_gpu_run_batch_from(const pire_gpu_scanner* sc, const uint8_t* d_corpus, const uint64_t* d_offsets, const uint32_t* d_order,
                            uint64_t fixed_len, uint64_t n, uint32_t flags, const uint32_t* d_start,
                            uint32_t* d_match_bits, uint32_t* d_accept_masks, uint32_t* d_state_idx, void* stream)
{
    int rc = CheckRunnable(sc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (flags & ~(PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END))
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_run_batch_from takes PIRE_GPU_RUN_BEGIN and PIRE_GPU_RUN_END only");
    if (n == 0)
        return PIRE_GPU_OK;
    if (!d_start)
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_run_batch_from needs n start states");
    if (!d_corpus && (d_offsets || fixed_len != 0))
        return Fail(PIRE_GPU_EINVAL, "null corpus with non-empty strings");
    if (d_order) {
        if (!d_offsets)
            return Fail(PIRE_GPU_EINVAL, "an order needs a CSR batch");
        return RunCsr(sc, d_corpus, d_offsets, d_order, n, flags, d_match_bits, d_accept_masks, d_state_idx, stream, d_start);
    }
    return RunBatch(sc, d_corpus, d_offsets, fixed_len, n, flags, d_start, d_match_bits, d_accept_masks, d_state_idx, stream);
}

int pire_gpu_run_pair_batch(const pire_gpu_scanner* sc1, const pire_gpu_scanner* sc2, const uint8_t* d_corpus,
                            const uint64_t* d_offsets, uint64_t fixed_len, uint64_t n, uint32_t flags, const uint32_t* d_start1,
                            const uint32_t* d_start2, uint32_t* d_match_bits1, uint32_t* d_accept_masks1, uint32_t* d_state_idx1,
                            uint32_t* d_match_bits2, uint32_t* d_accept_masks2, uint32_t* d_state_idx2, void* stream)
{
    int rc = CheckRunnable(sc1);
    if (rc == PIRE_GPU_OK)
        rc = CheckRunnable(sc2);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (sc1->device != sc2->device)
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_run_pair_batch needs two handles on one device");
    if (flags & ~(PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END))
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_run_pair_batch takes PIRE_GPU_RUN_BEGIN and PIRE_GPU_RUN_END only");
    if (n == 0)
        return PIRE_GPU_OK;
    if (!d_corpus && (d_offsets || fixed_len != 0))
        return Fail(PIRE_GPU_EINVAL, "null corpus with non-empty strings");
    if (n > (1ull << 40))
        return Fail(PIRE_GPU_EINVAL, "too many strings");
    if (!IsUniform(d_corpus, d_offsets, fixed_len)) {
        // not fused: each scanner's own batch launch, one after the other on the stream
        rc = RunBatch(sc1, d_corpus, d_offsets, fixed_len, n, flags, d_start1, d_match_bits1, d_accept_masks1, d_state_idx1, stream);
        if (rc != PIRE_GPU_OK)
            return rc;
        return RunBatch(sc2, d_corpus, d_offsets, fixed_len, n, flags, d_start2, d_match_bits2, d_accept_masks2, d_state_idx2, stream);
    }
    CUDA_TRY(cudaSetDevice(sc1->device));
    ScanArgs a[2];
    const pire_gpu_scanner* sc[2] = {sc1, sc2};
    const uint32_t* start[2] = {d_start1, d_start2};
    uint32_t* bits[2] = {d_match_bits1, d_match_bits2};
    uint32_t* masks[2] = {d_accept_masks1, d_accept_masks2};
    uint32_t* states[2] = {d_state_idx1, d_state_idx2};
    for (int k = 0; k < 2; ++k) {
        FillArgs(sc[k], &a[k], d_corpus, nullptr, fixed_len, n, flags);
        a[k].match_bits = bits[k];
        a[k].accept_masks = masks[k];
        a[k].state_idx = states[k];
        if (start[k])
            SetStarts(sc[k], &a[k], start[k], flags);
    }
    CUDA_TRY(LaunchPair(a[0], a[1], sc1->device, static_cast<cudaStream_t>(stream)));
    return PIRE_GPU_OK;
}

int pire_gpu_run_batch_ordered(const pire_gpu_scanner* sc, const uint8_t* d_corpus, const uint64_t* d_offsets,
                               const uint32_t* d_order, uint64_t n, uint32_t flags,
                               uint32_t* d_match_bits, uint32_t* d_accept_masks, uint32_t* d_state_idx, void* stream)
{
    if (n != 0 && !d_order)
        return Fail(PIRE_GPU_EINVAL, "ordered runs need corpus, CSR offsets and an order");
    return RunCsr(sc, d_corpus, d_offsets, d_order, n, flags, d_match_bits, d_accept_masks, d_state_idx, stream);
}

int pire_gpu_split_lines(const uint8_t* d_text, uint64_t n_bytes, uint64_t* d_line_offsets, uint64_t capacity,
                         uint64_t* n_lines, int device, void* stream)
{
    if (!n_lines || (n_bytes && !d_text))
        return Fail(PIRE_GPU_EINVAL, "null text or n_lines");
    CUDA_TRY(cudaSetDevice(device));
    uint64_t lines = 0;
    cudaError_t ce = SplitLines(d_text, n_bytes, d_line_offsets, capacity, &lines, static_cast<cudaStream_t>(stream));
    *n_lines = lines;
    if (ce == cudaErrorInvalidValue)
        return Fail(PIRE_GPU_EINVAL, "line offset buffer too small; *n_lines holds a sufficient capacity");
    if (ce != cudaSuccess)
        return FailCuda(ce, "pire_gpu_split_lines");
    return PIRE_GPU_OK;
}

int pire_gpu_run_lines(const pire_gpu_scanner* sc, const uint8_t* d_text, const uint64_t* d_line_offsets,
                       const uint32_t* d_order, uint64_t n_lines, uint32_t flags,
                       uint32_t* d_match_bits, uint32_t* d_accept_masks, uint32_t* d_state_idx, void* stream)
{
    return RunCsr(sc, d_text, d_line_offsets, d_order, n_lines, flags | PIRE_GPU_RUN_LINES, d_match_bits, d_accept_masks,
                  d_state_idx, stream);
}

int pire_gpu_run_pair_lines(const pire_gpu_scanner* sc1, const pire_gpu_scanner* sc2, const uint8_t* d_text,
                            const uint64_t* d_line_offsets, uint64_t n_lines, uint32_t flags, uint32_t* d_match_bits1,
                            uint32_t* d_accept_masks1, uint32_t* d_state_idx1, uint32_t* d_match_bits2, uint32_t* d_accept_masks2,
                            uint32_t* d_state_idx2, void* stream)
{
    int rc = CheckRunnable(sc1);
    if (rc == PIRE_GPU_OK)
        rc = CheckRunnable(sc2);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (sc1->device != sc2->device)
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_run_pair_lines needs two handles on one device");
    if (flags & ~(PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END | PIRE_GPU_RUN_LINES))
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_run_pair_lines takes PIRE_GPU_RUN_BEGIN, PIRE_GPU_RUN_END and PIRE_GPU_RUN_LINES only");
    if (n_lines == 0)
        return PIRE_GPU_OK;
    if (!d_text || !d_line_offsets)
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_run_pair_lines needs the text and its line offsets");
    if (n_lines >= (1ull << 31))
        return Fail(PIRE_GPU_EINVAL, "too many lines");
    CUDA_TRY(cudaSetDevice(sc1->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ScanArgs a[2];
    int variant[2];
    const pire_gpu_scanner* sc[2] = {sc1, sc2};
    uint32_t* bits[2] = {d_match_bits1, d_match_bits2};
    uint32_t* masks[2] = {d_accept_masks1, d_accept_masks2};
    uint32_t* states[2] = {d_state_idx1, d_state_idx2};
    for (int k = 0; k < 2; ++k) {
        FillArgs(sc[k], &a[k], d_text, d_line_offsets, 0, n_lines, flags | PIRE_GPU_RUN_LINES);
        a[k].match_bits = bits[k];
        a[k].accept_masks = masks[k];
        a[k].state_idx = states[k];
        variant[k] = (int) BatchVariant(sc[k], false, n_lines);
        // match bits are OR-ed into a zeroed bitmap, as pire_gpu_run_lines does
        if (bits[k])
            CUDA_TRY(cudaMemsetAsync(bits[k], 0, (size_t) ((n_lines + 31) / 32) * 4, st));
    }
    CUDA_TRY(LaunchPairLines(a[0], a[1], variant[0], variant[1], sc1->device, st));
    return PIRE_GPU_OK;
}

static int RunCsr(const pire_gpu_scanner* sc, const uint8_t* d_corpus, const uint64_t* d_offsets, const uint32_t* d_order,
                  uint64_t n, uint32_t flags, uint32_t* d_match_bits, uint32_t* d_accept_masks, uint32_t* d_state_idx,
                  void* stream, const uint32_t* d_start)
{
    int rc = CheckRunnable(sc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (flags & ~(PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END | PIRE_GPU_RUN_LINES))
        return Fail(PIRE_GPU_EINVAL, "unknown run flags");
    if (n == 0)
        return PIRE_GPU_OK;
    if (!d_corpus || !d_offsets)
        return Fail(PIRE_GPU_EINVAL, "CSR runs need a corpus and offsets");
    if (n >= (1ull << 31))
        return Fail(PIRE_GPU_EINVAL, "too many strings");
    CUDA_TRY(cudaSetDevice(sc->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ScanArgs a;
    FillArgs(sc, &a, d_corpus, d_offsets, 0, n, flags);
    a.order = d_order;
    a.match_bits = d_match_bits;
    a.accept_masks = d_accept_masks;
    a.state_idx = d_state_idx;
    unsigned int* counter = nullptr;
    cudaError_t ce = cudaSuccess;
    const bool split = d_order && !(flags & PIRE_GPU_RUN_LINES);
    if (d_order) {
        // length-binned: units are claimed longest-first, match bits are OR-ed into a zeroed bitmap; three words:
        // the generic kernel's unit counter, the split kernel's string counter, the number of strings it owns
        CUDA_TRY(ScratchAlloc(reinterpret_cast<void**>(&counter), 4 * sizeof(unsigned int), st));
        ce = cudaMemsetAsync(counter, 0, 4 * sizeof(unsigned int), st);
        if (ce == cudaSuccess && d_match_bits)
            ce = cudaMemsetAsync(d_match_bits, 0, (size_t) ((n + 31) / 32) * 4, st);
        a.work_counter = counter;
        if (split) {
            a.split_counter = counter + 1;
            a.split_count = counter + 2;
        }
    }
    const uint32_t variant = BatchVariant(sc, false, n);
    const LaunchPlan& plan = d_start ? sc->plan_from[variant][0] : sc->plan[variant][0];
    if (d_start)
        SetStarts(sc, &a, d_start, flags);
    if (split && ce == cudaSuccess)
        ce = LaunchSplit(a, (int) variant, sc->device, st);       // the long strings, one per warp; the rest below
    if ((flags & PIRE_GPU_RUN_LINES) && !d_order) {
        // lines of text: lanes pull lines dynamically and OR their match bits into a zeroed bitmap
        if (d_match_bits)
            ce = cudaMemsetAsync(d_match_bits, 0, (size_t) ((n + 31) / 32) * 4, st);
        if (ce == cudaSuccess)
            ce = LaunchLines(a, (int) variant, sc->device, st);
    } else if (ce == cudaSuccess)
        ce = LaunchScan(a, (int) variant, false, plan, st);
    if (counter)
        cudaFreeAsync(counter, st);
    if (ce != cudaSuccess)
        return FailCuda(ce, "pire_gpu_run_batch (CSR)");
    return PIRE_GPU_OK;
}

int pire_gpu_run_string(const pire_gpu_scanner* sc, const uint8_t* d_text, uint64_t n_bytes, uint32_t flags,
                        const uint32_t* d_start, uint32_t* d_match_bits, uint32_t* d_accept_masks, uint32_t* d_state_idx,
                        void* stream)
{
    int rc = CheckRunnable(sc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (flags & ~(PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END))
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_run_string takes PIRE_GPU_RUN_BEGIN and PIRE_GPU_RUN_END only");
    if (!d_text && n_bytes)
        return Fail(PIRE_GPU_EINVAL, "null text with n_bytes > 0");
    CUDA_TRY(cudaSetDevice(sc->device));
    ScanArgs a;
    FillArgs(sc, &a, d_text, nullptr, n_bytes, 1, flags);
    a.start_idx = d_start;
    a.new_of_old = sc->dev.new_of_old;
    a.states = sc->tab.states;
    a.with_begin = (flags & PIRE_GPU_RUN_BEGIN) ? 1 : 0;
    a.begin_class = sc->tab.begin_class;
    a.match_bits = d_match_bits;
    a.accept_masks = d_accept_masks;
    a.state_idx = d_state_idx;
    uint32_t variant = ResolveVariant(sc, false);
    if (variant == PIRE_GPU_VARIANT_PRIV)
        variant = PIRE_GPU_VARIANT_PLAIN;
    CUDA_TRY(LaunchString(a, (int) variant, sc->device, static_cast<cudaStream_t>(stream)));
    return PIRE_GPU_OK;
}

int pire_gpu_count_string(const pire_gpu_scanner* sc, const uint8_t* d_text, uint64_t n_bytes, uint32_t flags,
                          const uint32_t* d_start, uint64_t* d_counts, uint32_t* d_match_bits, uint32_t* d_state_idx, void* stream)
{
    int rc = CheckRunnable(sc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (flags & ~(PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END))
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_count_string takes PIRE_GPU_RUN_BEGIN and PIRE_GPU_RUN_END only");
    if (!d_counts)
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_count_string needs max(1, regexps) u64 counters");
    if (!d_text && n_bytes)
        return Fail(PIRE_GPU_EINVAL, "null text with n_bytes > 0");
    CUDA_TRY(cudaSetDevice(sc->device));
    ScanArgs a;
    FillArgs(sc, &a, d_text, nullptr, n_bytes, 1, flags);
    a.start_idx = d_start;
    a.new_of_old = sc->dev.new_of_old;
    a.states = sc->tab.states;
    a.with_begin = (flags & PIRE_GPU_RUN_BEGIN) ? 1 : 0;
    a.begin_class = sc->tab.begin_class;
    a.match_bits = d_match_bits;
    a.state_idx = d_state_idx;
    SetCounting(sc, &a, flags);
    a.counts64 = reinterpret_cast<unsigned long long*>(d_counts);
    a.count_rows = a.regexps <= kCountRowsMax ? 1 : 0;
    CUDA_TRY(LaunchCountString(a, sc->device, static_cast<cudaStream_t>(stream)));
    return PIRE_GPU_OK;
}

int pire_gpu_match_ends_string(const pire_gpu_scanner* sc, const uint8_t* d_text, uint64_t n_bytes, uint32_t flags,
                               const uint32_t* d_start, uint64_t base, uint64_t* d_ends, uint32_t* d_ids, uint64_t capacity,
                               uint64_t* d_found, uint32_t* d_match_bits, uint32_t* d_state_idx, void* stream)
{
    int rc = CheckRunnable(sc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (flags & ~(PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END))
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_match_ends_string takes PIRE_GPU_RUN_BEGIN and PIRE_GPU_RUN_END only");
    if (!d_found)
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_match_ends_string needs a device word for the number of entries");
    if (!d_text && n_bytes)
        return Fail(PIRE_GPU_EINVAL, "null text with n_bytes > 0");
    CUDA_TRY(cudaSetDevice(sc->device));
    ScanArgs a;
    FillArgs(sc, &a, d_text, nullptr, n_bytes, 1, flags);
    a.start_idx = d_start;
    a.new_of_old = sc->dev.new_of_old;
    a.states = sc->tab.states;
    a.match_bits = d_match_bits;
    a.state_idx = d_state_idx;
    SetCounting(sc, &a, flags);
    a.ends = d_ends;
    a.ids = d_ids;
    a.ends_capacity = capacity;
    a.found = reinterpret_cast<unsigned long long*>(d_found);
    a.ends_base = base;
    CUDA_TRY(LaunchMatchEndsString(a, sc->device, static_cast<cudaStream_t>(stream)));
    return PIRE_GPU_OK;
}

// Both match-starts entry points: the string form is a batch of one string whose window ends at base + n_bytes.
// lines: d_offsets are a text's lines (pire_gpu_match_starts_lines), each entry's window its own line.
static int MatchStarts(const pire_gpu_scanner* rsc, const uint8_t* d_corpus, const uint64_t* d_offsets, uint64_t fixed_len,
                       uint64_t n, const uint64_t* d_pos, uint64_t base, uint32_t flags, uint64_t max_back,
                       const uint32_t* d_strings, const uint64_t* d_ends, const uint32_t* d_ids, const uint64_t* d_first,
                       const uint64_t* d_found, uint64_t capacity, uint64_t* d_starts, uint8_t* d_open, void* stream,
                       bool lines = false)
{
    int rc = CheckRunnable(rsc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (flags & ~(PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END))
        return Fail(PIRE_GPU_EINVAL, "the match-starts calls take PIRE_GPU_RUN_BEGIN and PIRE_GPU_RUN_END only");
    if (!d_ends || !d_found || !d_starts)
        return Fail(PIRE_GPU_EINVAL, "the match-starts calls need d_ends, d_found and d_starts");
    if (!d_corpus && (d_offsets || fixed_len != 0))
        return Fail(PIRE_GPU_EINVAL, "null text with a non-empty window");
    if (n == 0 || capacity == 0)
        return PIRE_GPU_OK;
    if (n >= (1ull << 32))
        return Fail(PIRE_GPU_EINVAL, "too many strings: string indices are u32");
    CUDA_TRY(cudaSetDevice(rsc->device));
    ScanArgs a;
    FillArgs(rsc, &a, d_corpus, d_offsets, fixed_len, n, 0);
    a.flags = rsc->dev.flags;
    a.fin = rsc->dev.fin[0];                      // AcceptedRegexps of the state itself
    a.acc_begin = rsc->dev.acc_begin;
    a.acc_ids = rsc->dev.acc_ids;
    a.first_final_hot = rsc->tab.first_final_hot;
    a.initial = rsc->tab.initial;
    a.begin_class = rsc->tab.begin_class;
    a.end_class = rsc->tab.end_class;
    a.with_begin = (flags & PIRE_GPU_RUN_BEGIN) ? 1 : 0;
    a.with_end = (flags & PIRE_GPU_RUN_END) ? 1 : 0;
    a.live = rsc->dev.live;
    a.live_words = rsc->tab.live_words;
    a.window_end = d_pos;
    a.ends_base = base;
    a.max_back = max_back;
    a.entry_strings = d_strings;
    a.entry_ends = d_ends;
    a.entry_ids = d_ids;
    a.entries_first = reinterpret_cast<const unsigned long long*>(d_first);
    a.entries_found = reinterpret_cast<const unsigned long long*>(d_found);
    a.ends_capacity = capacity;
    a.match_starts = d_starts;
    a.match_open = d_open;
    a.trim = lines ? 1 : 0;
    CUDA_TRY(LaunchMatchStarts(a, rsc->device, static_cast<cudaStream_t>(stream)));
    return PIRE_GPU_OK;
}

int pire_gpu_match_starts_string(const pire_gpu_scanner* rsc, const uint8_t* d_text, uint64_t n_bytes, uint64_t base,
                                 uint32_t flags, uint64_t max_back, const uint64_t* d_ends, const uint32_t* d_ids,
                                 const uint64_t* d_first, const uint64_t* d_found, uint64_t capacity, uint64_t* d_starts,
                                 uint8_t* d_open, void* stream)
{
    return MatchStarts(rsc, d_text, nullptr, n_bytes, 1, nullptr, base, flags, max_back, nullptr, d_ends, d_ids, d_first, d_found,
                       capacity, d_starts, d_open, stream);
}

int pire_gpu_match_starts_batch(const pire_gpu_scanner* rsc, const uint8_t* d_corpus, const uint64_t* d_offsets,
                                uint64_t fixed_len, uint64_t n, const uint64_t* d_pos, uint32_t flags, uint64_t max_back,
                                const uint32_t* d_strings, const uint64_t* d_ends, const uint32_t* d_ids,
                                const uint64_t* d_first, const uint64_t* d_found, uint64_t capacity,
                                uint64_t* d_starts, uint8_t* d_open, void* stream)
{
    return MatchStarts(rsc, d_corpus, d_offsets, fixed_len, n, d_pos, 0, flags, max_back, d_strings, d_ends, d_ids, d_first,
                       d_found, capacity, d_starts, d_open, stream);
}

int pire_gpu_match_starts_lines(const pire_gpu_scanner* rsc, const uint8_t* d_text, const uint64_t* d_line_offsets,
                                uint64_t n_lines, uint32_t flags, uint64_t max_back, const uint32_t* d_lines,
                                const uint64_t* d_ends, const uint32_t* d_ids, const uint64_t* d_first, const uint64_t* d_found,
                                uint64_t capacity, uint64_t* d_starts, uint8_t* d_open, void* stream)
{
    int rc = CheckRunnable(rsc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (!d_line_offsets || !d_lines)
        return Fail(PIRE_GPU_EINVAL, "pire_gpu_match_starts_lines needs the line offsets and d_lines");
    return MatchStarts(rsc, d_text, d_line_offsets, 0, n_lines, nullptr, 0, flags & ~PIRE_GPU_RUN_LINES, max_back, d_lines,
                       d_ends, d_ids, d_first, d_found, capacity, d_starts, d_open, stream, true);
}

int pire_gpu_scanner_tune(pire_gpu_scanner* sc, const uint8_t* d_corpus, const uint64_t* d_offsets,
                          uint64_t fixed_len, uint64_t n_sample, uint32_t flags, void* stream)
{
    int rc = CheckRunnable(sc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (n_sample == 0)
        return PIRE_GPU_OK;
    CUDA_TRY(cudaSetDevice(sc->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    unsigned long long* d_visits = nullptr;
    const size_t bytes = (size_t) sc->tab.states * sizeof(unsigned long long);
    CUDA_TRY(cudaMalloc(&d_visits, bytes));
    cudaError_t ce = cudaMemsetAsync(d_visits, 0, bytes, st);
    ScanArgs a;
    FillArgs(sc, &a, d_corpus, d_offsets, fixed_len, n_sample, flags);
    a.visits = d_visits;
    if (ce == cudaSuccess)
        ce = LaunchVisitCount(a, st);
    std::vector<unsigned long long> by_new(sc->tab.states);
    if (ce == cudaSuccess)
        ce = cudaMemcpyAsync(by_new.data(), d_visits, bytes, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess)
        ce = cudaStreamSynchronize(st);
    cudaFree(d_visits);
    if (ce != cudaSuccess)
        return FailCuda(ce, "pire_gpu_scanner_tune");
    std::vector<uint64_t> by_old(sc->dfa.states, 0);
    for (uint32_t ns = 0; ns < sc->tab.states; ++ns)
        by_old[sc->tab.old_of_new[ns]] = by_new[ns];
    try {
        sc->hot_order = HotOrderFromCounts(sc->dfa, by_old);
    } catch (const std::exception& e) {
        return Fail(PIRE_GPU_EINVAL, std::string("pire_gpu_scanner_tune: ") + e.what());
    }
    uint64_t steps = 0, in_final = 0;
    for (uint32_t s = 0; s < sc->dfa.states; ++s) {
        steps += by_old[s];
        if (sc->dfa.Final(s))
            in_final += by_old[s];
    }
    sc->final_share = steps ? (double) in_final / (double) steps : 0.0;
    sc->tuned = true;
    try {
        Rebuild(sc);
    } catch (const std::exception& e) {
        return Fail(PIRE_GPU_EINVAL, std::string("pire_gpu_scanner_tune: ") + e.what());
    }
    return Upload(sc);
}

int pire_gpu_scanner_autoselect(pire_gpu_scanner* sc, const uint8_t* d_corpus, const uint64_t* d_offsets,
                                uint64_t fixed_len, uint64_t n, uint32_t flags, void* stream, float* ms_out)
{
    int rc = CheckRunnable(sc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (ms_out)
        for (int v = 0; v < PIRE_GPU_VARIANT_SLOTS; ++v)
            ms_out[v] = 0.f;
    if (n == 0)
        return PIRE_GPU_OK;
    CUDA_TRY(cudaSetDevice(sc->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool uniform = IsUniform(d_corpus, d_offsets, fixed_len);
    uint32_t* scratch = nullptr;
    const size_t words = (size_t) ((n + 31) / 32);
    CUDA_TRY(cudaMalloc(&scratch, (words + n) * 4));
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    cudaError_t ce = cudaEventCreate(&e0);
    if (ce == cudaSuccess)
        ce = cudaEventCreate(&e1);
    // ragged CSR batches are timed the way they are run by the host entry point and the benchmark: binned by length
    uint32_t* order = nullptr;
    if (ce == cudaSuccess && d_offsets && !(flags & PIRE_GPU_RUN_LINES) && n >= 64 && n < (1ull << 31)) {
        ce = cudaMalloc(&order, (size_t) n * 4);
        if (ce == cudaSuccess)
            ce = LengthOrder(d_offsets, n, order, st);
    }
    const uint32_t saved = sc->variant;
    uint32_t best = 0;
    float best_ms = 0.f;
    for (uint32_t v = PIRE_GPU_VARIANT_PLAIN; v <= PIRE_GPU_VARIANT_LOOK_RING1 && ce == cudaSuccess; ++v) {
        if (v == PIRE_GPU_VARIANT_PRIV && !(uniform && sc->priv_ok))
            continue;
        if (v >= PIRE_GPU_VARIANT_LOOK && !sc->tab.look_ok)
            continue;
        if ((v == PIRE_GPU_VARIANT_LOOK64 || v == PIRE_GPU_VARIANT_LOOK1 || v == PIRE_GPU_VARIANT_LOOK_RING1) && !uniform)
            continue;               // CSR batches have one look-ahead kernel
        sc->variant = v;
        float ms = 0.f;
        for (int rep = 0; rep < 2 && rc == PIRE_GPU_OK; ++rep) {      // first launch warms, second is timed
            cudaEventRecord(e0, st);
            rc = order ? pire_gpu_run_batch_ordered(sc, d_corpus, d_offsets, order, n, flags, scratch, scratch + words, nullptr, st)
                       : pire_gpu_run_batch(sc, d_corpus, d_offsets, fixed_len, n, flags, scratch, scratch + words, nullptr, st);
            cudaEventRecord(e1, st);
            ce = cudaEventSynchronize(e1);
            if (ce == cudaSuccess)
                ce = cudaEventElapsedTime(&ms, e0, e1);
        }
        if (rc != PIRE_GPU_OK)
            break;
        if (ms_out)
            ms_out[v] = ms;
        if (best == 0 || ms < best_ms) {
            best = v;
            best_ms = ms;
        }
    }
    sc->variant = saved;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaFree(scratch);
    cudaFree(order);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (ce != cudaSuccess)
        return FailCuda(ce, "pire_gpu_scanner_autoselect");
    sc->auto_choice[uniform ? 1 : 0] = best;
    return PIRE_GPU_OK;
}

uint64_t pire_gpu_launch_count(void) { return KernelLaunchCount(); }

uint32_t pire_gpu_initial(const pire_gpu_scanner* sc) { return sc ? sc->dfa.initial : 0; }

uint32_t pire_gpu_next(const pire_gpu_scanner* sc, uint32_t state, uint32_t ch)
{
    if (!sc || state >= sc->dfa.states || ch >= kMaxCharUnaligned)
        return 0;
    return sc->dfa.Next(state, ch);
}

int pire_gpu_final(const pire_gpu_scanner* sc, uint32_t state)
{
    return sc && state < sc->dfa.states && sc->dfa.Final(state);
}

int pire_gpu_dead(const pire_gpu_scanner* sc, uint32_t state)
{
    return sc && state < sc->dfa.states && sc->dfa.Dead(state);
}

size_t pire_gpu_accepted_regexps(const pire_gpu_scanner* sc, uint32_t state, uint32_t* ids, size_t cap)
{
    if (!sc || state >= sc->dfa.states)
        return 0;
    size_t k = 0;
    for (uint32_t at = sc->dfa.acc_begin[state]; at < sc->dfa.acc_begin[state + 1]; ++at, ++k)
        if (ids && k < cap)
            ids[k] = sc->dfa.acc_ids[at];
    return k;
}

static int FillSynthParams(const pire_gpu_synth* spec, SynthParams* p)
{
    if (!spec)
        return Fail(PIRE_GPU_EINVAL, "null synth spec");
    if (spec->string_len == 0 || spec->string_len % 16 != 0)
        return Fail(PIRE_GPU_EINVAL, "string_len must be a positive multiple of 16");
    if (spec->kind != 0)
        return Fail(PIRE_GPU_EUNSUPPORTED, "unknown synthetic corpus kind");
    if (spec->n_plants > (uint32_t) kMaxPlants)
        return Fail(PIRE_GPU_EINVAL, "too many plants");
    std::memset(p, 0, sizeof(*p));
    p->seed = spec->seed;
    p->first_string = spec->first_string;
    p->n_strings = spec->n_strings;
    p->string_len = spec->string_len;
    p->plant_every = spec->plant_every;
    p->n_plants = spec->n_plants;
    p->tail = spec->tail;
    uint32_t at = 0;
    const char* lit = spec->plants;
    const char* lim = spec->plants + spec->plants_bytes;
    for (uint32_t i = 0; i < spec->n_plants; ++i) {
        if (lit >= lim)
            return Fail(PIRE_GPU_EINVAL, "plants buffer shorter than n_plants literals");
        size_t len = strnlen(lit, (size_t) (lim - lit));
        if (lit + len >= lim)
            return Fail(PIRE_GPU_EINVAL, "plants buffer not NUL-terminated");
        p->plant_off[i] = at;
        p->plant_mode[i] = lit[0] == '^' ? 1 : lit[0] == '$' ? 2 : 0;
        at += (uint32_t) (len - (p->plant_mode[i] ? 1 : 0));
        lit += len + 1;
    }
    p->plant_off[spec->n_plants] = at;
    return PIRE_GPU_OK;
}

// plants without the separating NULs, indexable by plant_off
static std::string PackPlants(const pire_gpu_synth* spec)
{
    std::string packed;
    const char* q = spec->plants;
    for (uint32_t i = 0; i < spec->n_plants; ++i) {
        size_t len = std::strlen(q);
        size_t skip = (q[0] == '^' || q[0] == '$') ? 1 : 0;
        packed.append(q + skip, len - skip);
        q += len + 1;
    }
    return packed;
}

int pire_gpu_synth_fill_device(const pire_gpu_synth* spec, uint8_t* d_corpus, int device, void* stream)
{
    SynthParams p;
    int rc = FillSynthParams(spec, &p);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (!d_corpus)
        return Fail(PIRE_GPU_EINVAL, "null device corpus");
    CUDA_TRY(cudaSetDevice(device));
    std::string packed = PackPlants(spec);
    char* d_plants = nullptr;
    CUDA_TRY(cudaMalloc(&d_plants, packed.size() + 16));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t ce = cudaMemcpyAsync(d_plants, packed.data(), packed.size(), cudaMemcpyHostToDevice, st);
    if (ce == cudaSuccess)
        ce = LaunchSynth(p, d_plants, d_corpus, st);
    if (ce == cudaSuccess)
        ce = cudaStreamSynchronize(st);
    cudaFree(d_plants);
    if (ce != cudaSuccess)
        return FailCuda(ce, "pire_gpu_synth_fill_device");
    return PIRE_GPU_OK;
}

int pire_gpu_synth_fill_host(const pire_gpu_synth* spec, uint8_t* corpus, uint64_t first, uint64_t count)
{
    SynthParams p;
    int rc = FillSynthParams(spec, &p);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (!corpus)
        return Fail(PIRE_GPU_EINVAL, "null corpus");
    std::string packed = PackPlants(spec);
    const uint32_t words = p.string_len / 8;
    for (uint64_t k = 0; k < count; ++k) {
        const uint64_t gi = p.first_string + first + k;
        uint8_t* dst = corpus + k * (uint64_t) p.string_len;
        for (uint32_t w = 0; w < words; ++w) {
            uint64_t v = SynthWord(p.seed, gi, w, words);
            std::memcpy(dst + (size_t) w * 8, &v, 8);
        }
        uint32_t off = 0;
        int id = SynthPlant(p, gi, &off);
        if (id >= 0) {
            std::memcpy(dst + off, packed.data() + p.plant_off[id], p.plant_off[id + 1] - p.plant_off[id]);
            if (p.tail && p.plant_mode[id] == 0)
                dst[p.string_len - 1] = (uint8_t) p.tail;
        }
    }
    return PIRE_GPU_OK;
}

int pire_gpu_synth_fill_host_indexed(const pire_gpu_synth* spec, uint8_t* corpus, const uint64_t* indices, uint64_t count)
{
    SynthParams p;
    int rc = FillSynthParams(spec, &p);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (count && (!corpus || !indices))
        return Fail(PIRE_GPU_EINVAL, "null corpus or indices");
    std::string packed = PackPlants(spec);
    const uint32_t words = p.string_len / 8;
    for (uint64_t k = 0; k < count; ++k) {
        const uint64_t gi = p.first_string + indices[k];
        uint8_t* dst = corpus + k * (uint64_t) p.string_len;
        for (uint32_t w = 0; w < words; ++w) {
            uint64_t v = SynthWord(p.seed, gi, w, words);
            std::memcpy(dst + (size_t) w * 8, &v, 8);
        }
        uint32_t off = 0;
        int id = SynthPlant(p, gi, &off);
        if (id >= 0) {
            std::memcpy(dst + off, packed.data() + p.plant_off[id], p.plant_off[id + 1] - p.plant_off[id]);
            if (p.tail && p.plant_mode[id] == 0)
                dst[p.string_len - 1] = (uint8_t) p.tail;
        }
    }
    return PIRE_GPU_OK;
}

int pire_gpu_synth_mixed_lengths_device(uint64_t seed, uint64_t first_string, uint64_t n, uint64_t* d_lengths, int device, void* stream)
{
    if (!d_lengths && n)
        return Fail(PIRE_GPU_EINVAL, "null lengths");
    CUDA_TRY(cudaSetDevice(device));
    CUDA_TRY(LaunchSynthMixedLengths(seed, first_string, n, d_lengths, static_cast<cudaStream_t>(stream)));
    return PIRE_GPU_OK;
}

int pire_gpu_synth_mixed_lengths_host(uint64_t seed, uint64_t first_string, uint64_t n, uint64_t* lengths)
{
    if (!lengths && n)
        return Fail(PIRE_GPU_EINVAL, "null lengths");
    for (uint64_t i = 0; i < n; ++i)
        lengths[i] = SynthMixedLength(seed, first_string + i);
    return PIRE_GPU_OK;
}

int pire_gpu_synth_mixed_fill_device(uint64_t seed, uint32_t plant_every, uint64_t first_string, uint64_t n,
                                     const uint64_t* d_offsets, uint8_t* d_corpus, int device, void* stream)
{
    if (n && (!d_offsets || !d_corpus))
        return Fail(PIRE_GPU_EINVAL, "null offsets or corpus");
    CUDA_TRY(cudaSetDevice(device));
    CUDA_TRY(LaunchSynthMixedFill(seed, plant_every, first_string, n, d_offsets, d_corpus, static_cast<cudaStream_t>(stream)));
    return PIRE_GPU_OK;
}

int pire_gpu_synth_mixed_fill_host(uint64_t seed, uint32_t plant_every, uint64_t first_string, uint64_t n,
                                   const uint64_t* offsets, uint8_t* corpus)
{
    if (n && (!offsets || !corpus))
        return Fail(PIRE_GPU_EINVAL, "null offsets or corpus");
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t len = (uint32_t) (offsets[i + 1] - offsets[i]);
        for (uint32_t cell = 0; cell < len / 4; ++cell) {
            uint32_t v = SynthMixedCellPlanted(seed, plant_every, first_string + i, len, cell);
            std::memcpy(corpus + offsets[i] + (size_t) cell * 4, &v, 4);
        }
    }
    return PIRE_GPU_OK;
}

const char* pire_gpu_last_error(void) { return g_error.c_str(); }

const char* pire_gpu_version(void) { return "pire-b200 0.1 (sm_90a)"; }

} // extern "C"
