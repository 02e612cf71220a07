// capi_host.cu -- pire_gpu_run_batch_host: the caller the reference actually has.
//
// Pire::Runner(sc).Begin().Run(ptr, len).End() (run.h:271-275,:365-392) takes a plain `const char*` in pageable host
// memory (samples/pigrep/pigrep.cpp:38-45 hands it std::getline's buffer).  This entry point serves that caller for a
// whole batch: the corpus is cut into chunks of whole 32-string units and streamed through a small ring of device
// slots, so that
//   * the host->device copy of chunk k+1 overlaps the scan of chunk k and the device->host copy of its results,
//   * pageable input is staged through the library's own pinned buffers by a few copy threads (a cudaMemcpyAsync
//     from pageable memory is a synchronous, driver-staged copy at a fraction of the link rate); pinned or
//     registered input is DMA-ed straight from the caller's buffer,
//   * the device never holds more than the ring (corpora larger than HBM stream through),
//   * two threads calling on the same handle each take their own workspace and run concurrently.
// Results are identical to pire_gpu_run_batch on the resident corpus: chunk boundaries are multiples of 32
// strings, so bitmap words never straddle chunks.
#include "capi_internal.hpp"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <thread>

#include "stage_copy.hpp"

using namespace pire_b200;

namespace pire_b200 {

namespace {

// A few threads that copy slices of one buffer; the calling thread takes part.
class CopyPool {
public:
    explicit CopyPool(unsigned helpers)
    {
        for (unsigned i = 0; i < helpers; ++i)
            threads_.emplace_back([this] { Work(); });
    }
    ~CopyPool()
    {
        {
            std::lock_guard<std::mutex> lock(mu_);
            quit_ = true;
        }
        cv_.notify_all();
        for (std::thread& t : threads_)
            t.join();
    }
    void Copy(uint8_t* dst, const uint8_t* src, size_t bytes)
    {
        constexpr size_t kPiece = 2u << 20;
        if (threads_.empty() || bytes < 2 * kPiece) {
            StageCopy(dst, src, bytes);
            return;
        }
        {
            std::lock_guard<std::mutex> lock(mu_);
            dst_ = dst;
            src_ = src;
            bytes_ = bytes;
            pieces_ = (bytes + kPiece - 1) / kPiece;
            next_ = 0;
            left_ = pieces_;
            ++generation_;
        }
        cv_.notify_all();
        Drain();
        std::unique_lock<std::mutex> lock(mu_);
        done_.wait(lock, [this] { return left_ == 0; });
    }

private:
    // A piece is claimed under the lock, together with the buffers it belongs to: a helper still on its way out of
    // the previous copy cannot take a piece number from one copy and the buffers or the count of the next, so every
    // piece is counted off exactly once and Copy returns only when all of them have landed.
    void Drain()
    {
        constexpr size_t kPiece = 2u << 20;
        std::unique_lock<std::mutex> lock(mu_);
        while (next_ < pieces_) {
            const size_t at = next_++ * kPiece;
            uint8_t* dst = dst_ + at;
            const uint8_t* src = src_ + at;
            const size_t len = std::min(kPiece, bytes_ - at);
            lock.unlock();
            StageCopy(dst, src, len);
            lock.lock();
            if (--left_ == 0)
                done_.notify_all();
        }
    }
    void Work()
    {
        uint64_t seen = 0;
        for (;;) {
            {
                std::unique_lock<std::mutex> lock(mu_);
                cv_.wait(lock, [&] { return quit_ || generation_ != seen; });
                if (quit_)
                    return;
                seen = generation_;
            }
            Drain();
        }
    }
    std::vector<std::thread> threads_;
    std::mutex mu_;
    std::condition_variable cv_, done_;
    bool quit_ = false;
    uint64_t generation_ = 0;
    uint8_t* dst_ = nullptr;
    const uint8_t* src_ = nullptr;
    size_t bytes_ = 0, pieces_ = 0, next_ = 0, left_ = 0;
};

size_t EnvSize(const char* name, size_t fallback)
{
    const char* env = getenv(name);
    if (!env || !*env)
        return fallback;
    const long v = atol(env);
    return v > 0 ? (size_t) v : fallback;
}

bool IsPinned(const void* p)
{
    if (!p)
        return true;
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) {
        (void) cudaGetLastError();
        return false;
    }
    return attr.type == cudaMemoryTypeHost || attr.type == cudaMemoryTypeManaged;
}

} // namespace

constexpr int kHostSlots = 3;

struct HostSlot {
    uint8_t* h_in = nullptr;
    size_t h_in_bytes = 0;
    uint8_t* d_in = nullptr;
    size_t d_in_bytes = 0;
    // capacities are kept per buffer: an allocation that fails leaves ITS capacity at zero, so the next call allocates
    // again instead of trusting a pointer that is gone
    uint64_t* h_off = nullptr;
    size_t h_off_cap = 0;         // entries
    uint64_t* d_off = nullptr;
    size_t off_cap = 0;           // entries
    uint32_t* h_out = nullptr;
    size_t h_out_cap = 0;         // words
    uint32_t* d_out = nullptr;
    size_t out_cap = 0;           // words
    uint32_t* d_order = nullptr;
    size_t order_cap = 0;
    cudaEvent_t copied = nullptr, done = nullptr;
    // results waiting in h_out for the caller's arrays
    bool pending = false;
    uint64_t first = 0, count = 0;
};

struct HostWorkspace {
    cudaStream_t copy = nullptr, run = nullptr;
    HostSlot slot[kHostSlots];
    CopyPool* pool = nullptr;

    ~HostWorkspace()
    {
        delete pool;
        for (HostSlot& s : slot) {
            cudaFreeHost(s.h_in);
            cudaFree(s.d_in);
            cudaFreeHost(s.h_off);
            cudaFree(s.d_off);
            cudaFreeHost(s.h_out);
            cudaFree(s.d_out);
            cudaFree(s.d_order);
            if (s.copied)
                cudaEventDestroy(s.copied);
            if (s.done)
                cudaEventDestroy(s.done);
        }
        if (copy)
            cudaStreamDestroy(copy);
        if (run)
            cudaStreamDestroy(run);
    }
};

void FreeHostWorkspaces(pire_gpu_scanner* sc)
{
    std::lock_guard<std::mutex> lock(sc->ws_mutex);
    for (HostWorkspace* ws : sc->ws_free)
        delete ws;
    sc->ws_free.clear();
}

namespace {

template <class T>
cudaError_t GrowDevice(T** p, size_t* cap, size_t want)
{
    if (*cap >= want)
        return cudaSuccess;
    cudaFree(*p);
    *p = nullptr;
    *cap = 0;
    cudaError_t err = cudaMalloc(p, want * sizeof(T));
    if (err == cudaSuccess)
        *cap = want;
    return err;
}

template <class T>
cudaError_t GrowPinned(T** p, size_t* cap, size_t want)
{
    if (*cap >= want)
        return cudaSuccess;
    cudaFreeHost(*p);
    *p = nullptr;
    *cap = 0;
    cudaError_t err = cudaHostAlloc(p, want * sizeof(T), cudaHostAllocDefault);
    if (err == cudaSuccess)
        *cap = want;
    return err;
}

struct Caller {
    const uint8_t* corpus;
    const uint64_t* offsets;
    uint64_t fixed_len, n;
    uint32_t* match_bits;
    uint32_t* accept_masks;
    uint32_t* state_idx;
};

// the results of a finished chunk: out of the pinned slot into the caller's arrays
void CopyOut(const Caller& c, HostSlot& s)
{
    if (!s.pending)
        return;
    const size_t words = (size_t) ((s.count + 31) / 32);
    const uint32_t* at = s.h_out;
    if (c.match_bits) {
        std::memcpy(c.match_bits + s.first / 32, at, words * 4);
        at += words;
    }
    if (c.accept_masks) {
        std::memcpy(c.accept_masks + s.first, at, (size_t) s.count * 4);
        at += s.count;
    }
    if (c.state_idx)
        std::memcpy(c.state_idx + s.first, at, (size_t) s.count * 4);
    s.pending = false;
}

int RunStreamed(const pire_gpu_scanner* sc, HostWorkspace* ws, const Caller& c, uint64_t corpus_bytes, uint32_t flags)
{
    if (!ws->copy)
        CUDA_TRY(cudaStreamCreateWithFlags(&ws->copy, cudaStreamNonBlocking));
    if (!ws->run)
        CUDA_TRY(cudaStreamCreateWithFlags(&ws->run, cudaStreamNonBlocking));
    for (HostSlot& s : ws->slot) {
        if (!s.copied)
            CUDA_TRY(cudaEventCreateWithFlags(&s.copied, cudaEventDisableTiming));
        if (!s.done)
            CUDA_TRY(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
        s.pending = false;
    }
    const bool pinned_in = IsPinned(c.corpus) && !getenv("PIRE_B200_HOST_FORCE_STAGING");
    if (!pinned_in && !ws->pool) {
        unsigned hw = std::thread::hardware_concurrency();
        size_t threads = EnvSize("PIRE_B200_HOST_THREADS", std::min<size_t>(8, std::max<unsigned>(1, hw / 4)));
        ws->pool = new CopyPool((unsigned) (threads > 1 ? threads - 1 : 0));
    }
    const size_t chunk_bytes = EnvSize("PIRE_B200_HOST_CHUNK_MB", 64) << 20;
    const bool csr = c.offsets != nullptr;
    const bool lines = csr && (flags & PIRE_GPU_RUN_LINES);
    const int outputs = (c.match_bits ? 1 : 0) + (c.accept_masks ? 1 : 0) + (c.state_idx ? 1 : 0);

    uint64_t first = 0;
    for (uint64_t k = 0; first < c.n; ++k) {
        HostSlot& s = ws->slot[k % kHostSlots];
        // the slot's previous chunk: wait for it and hand its results to the caller
        if (s.pending) {
            CUDA_TRY(cudaEventSynchronize(s.done));
            CopyOut(c, s);
        }
        // this chunk: whole 32-string units, about chunk_bytes of corpus
        uint64_t count;
        uint64_t byte_lo, byte_hi, copy_hi;
        if (csr) {
            byte_lo = c.offsets[first];
            uint64_t last = first;
            do {
                last = std::min<uint64_t>(c.n, last + 32);
            } while (last < c.n && c.offsets[std::min<uint64_t>(c.n, last + 32)] - byte_lo <= chunk_bytes);
            count = last - first;
            byte_hi = c.offsets[last];
            // the batch's last line ends at a separator that may be the virtual one after the text
            // (pire_gpu_split_lines); no kernel reads that byte, so the copy stops short of it
            copy_hi = lines && last == c.n ? byte_hi - 1 : byte_hi;
            if (byte_hi < byte_lo || copy_hi < byte_lo || copy_hi > corpus_bytes)
                return Fail(PIRE_GPU_EINVAL, "offsets are not ascending or run past corpus_bytes");
        } else {
            const uint64_t per = c.fixed_len ? std::max<uint64_t>(32, chunk_bytes / c.fixed_len / 32 * 32) : c.n;
            count = std::min<uint64_t>(per, c.n - first);
            byte_lo = first * c.fixed_len;
            byte_hi = byte_lo + count * c.fixed_len;
            copy_hi = byte_hi;
        }
        const size_t bytes = (size_t) (copy_hi - byte_lo);
        const size_t words = (size_t) ((count + 31) / 32);
        const size_t out_words = (c.match_bits ? words : 0) + (size_t) ((c.accept_masks ? 1 : 0) + (c.state_idx ? 1 : 0)) * count;

        CUDA_TRY(GrowDevice(&s.d_in, &s.d_in_bytes, bytes + 64));
        if (out_words) {
            CUDA_TRY(GrowPinned(&s.h_out, &s.h_out_cap, out_words));
            CUDA_TRY(GrowDevice(&s.d_out, &s.out_cap, out_words));
        }
        const uint8_t* dma_src = c.corpus ? c.corpus + byte_lo : nullptr;
        if (!pinned_in && bytes) {
            CUDA_TRY(GrowPinned(&s.h_in, &s.h_in_bytes, bytes));
            ws->pool->Copy(s.h_in, c.corpus + byte_lo, bytes);
            dma_src = s.h_in;
        }
        if (csr) {
            CUDA_TRY(GrowPinned(&s.h_off, &s.h_off_cap, (size_t) count + 1));
            CUDA_TRY(GrowDevice(&s.d_off, &s.off_cap, (size_t) count + 1));
            uint64_t prev = byte_lo;
            for (uint64_t i = 0; i <= count; ++i) {
                const uint64_t o = c.offsets[first + i];
                if (o < prev)
                    return Fail(PIRE_GPU_EINVAL, "offsets are not ascending");
                prev = o;
                s.h_off[i] = o - byte_lo;          // the chunk's own CSR, rebased to its slot
            }
        }
        if (bytes)
            CUDA_TRY(cudaMemcpyAsync(s.d_in, dma_src, bytes, cudaMemcpyHostToDevice, ws->copy));
        if (csr)
            CUDA_TRY(cudaMemcpyAsync(s.d_off, s.h_off, (size_t) (count + 1) * 8, cudaMemcpyHostToDevice, ws->copy));
        CUDA_TRY(cudaEventRecord(s.copied, ws->copy));
        CUDA_TRY(cudaStreamWaitEvent(ws->run, s.copied, 0));

        uint32_t* d_bits = c.match_bits ? s.d_out : nullptr;
        uint32_t* d_masks = c.accept_masks ? s.d_out + (c.match_bits ? words : 0) : nullptr;
        uint32_t* d_states = c.state_idx ? s.d_out + (c.match_bits ? words : 0) + (c.accept_masks ? count : 0) : nullptr;
        int rc;
        const bool binned = csr && count >= 64 && count < (1ull << 31) && !(flags & PIRE_GPU_RUN_LINES);
        if (binned) {
            // strings of unknown, unequal lengths: bin them so that a warp's lanes finish together
            CUDA_TRY(GrowDevice(&s.d_order, &s.order_cap, (size_t) count));
            CUDA_TRY(LengthOrder(s.d_off, count, s.d_order, ws->run));
            rc = pire_gpu_run_batch_ordered(sc, s.d_in, s.d_off, s.d_order, count, flags, d_bits, d_masks, d_states, ws->run);
        } else if (csr && (flags & PIRE_GPU_RUN_LINES)) {
            rc = pire_gpu_run_lines(sc, s.d_in, s.d_off, nullptr, count, flags, d_bits, d_masks, d_states, ws->run);
        } else {
            rc = pire_gpu_run_batch(sc, s.d_in, csr ? s.d_off : nullptr, c.fixed_len, count, flags, d_bits, d_masks, d_states, ws->run);
        }
        if (rc != PIRE_GPU_OK)
            return rc;
        if (outputs)
            CUDA_TRY(cudaMemcpyAsync(s.h_out, s.d_out, out_words * 4, cudaMemcpyDeviceToHost, ws->run));
        CUDA_TRY(cudaEventRecord(s.done, ws->run));
        s.pending = true;
        s.first = first;
        s.count = count;
        first += count;
    }
    for (HostSlot& s : ws->slot)
        if (s.pending) {
            CUDA_TRY(cudaEventSynchronize(s.done));
            CopyOut(c, s);
        }
    return PIRE_GPU_OK;
}

} // namespace

} // namespace pire_b200

extern "C" int pire_gpu_run_batch_host(const pire_gpu_scanner* csc, const uint8_t* corpus, uint64_t corpus_bytes,
                                       const uint64_t* offsets, uint64_t fixed_len, uint64_t n, uint32_t flags,
                                       uint32_t* match_bits, uint32_t* accept_masks, uint32_t* state_idx)
{
    int rc = CheckRunnable(csc);
    if (rc != PIRE_GPU_OK)
        return rc;
    if (flags & ~(PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END | PIRE_GPU_RUN_LINES))
        return Fail(PIRE_GPU_EINVAL, "unknown run flags");
    if (n == 0)
        return PIRE_GPU_OK;
    if (n > (1ull << 40))
        return Fail(PIRE_GPU_EINVAL, "too many strings");
    if (!corpus && corpus_bytes != 0)
        return Fail(PIRE_GPU_EINVAL, "null corpus with corpus_bytes != 0");
    if (offsets) {
        // a line batch needs the text up to its last separator, and a last line without '\n' has a virtual one at
        // offsets[n] - 1 == the text's size
        const uint64_t end = offsets[n] - ((flags & PIRE_GPU_RUN_LINES) ? 1 : 0);
        if (end > corpus_bytes || offsets[0] > end)
            return Fail(PIRE_GPU_EINVAL, "offsets run past corpus_bytes");
    } else if (fixed_len != 0 && (corpus_bytes / fixed_len < n)) {
        return Fail(PIRE_GPU_EINVAL, "n * fixed_len exceeds corpus_bytes");
    }
    pire_gpu_scanner* sc = const_cast<pire_gpu_scanner*>(csc);      // the workspace list is the handle's only mutable part
    CUDA_TRY(cudaSetDevice(sc->device));
    HostWorkspace* ws = nullptr;
    {
        std::lock_guard<std::mutex> lock(sc->ws_mutex);
        if (!sc->ws_free.empty()) {
            ws = sc->ws_free.back();
            sc->ws_free.pop_back();
        }
    }
    if (!ws)
        ws = new (std::nothrow) HostWorkspace;
    if (!ws)
        return Fail(PIRE_GPU_EINVAL, "out of memory");
    Caller c{corpus, offsets, fixed_len, n, match_bits, accept_masks, state_idx};
    try {
        rc = RunStreamed(sc, ws, c, corpus_bytes, flags);
    } catch (const std::exception& e) {
        rc = Fail(PIRE_GPU_EINVAL, std::string("pire_gpu_run_batch_host: ") + e.what());
    }
    if (rc != PIRE_GPU_OK) {
        // leave nothing in flight that still points at the caller's buffers
        if (ws->copy)
            cudaStreamSynchronize(ws->copy);
        if (ws->run)
            cudaStreamSynchronize(ws->run);
        (void) cudaGetLastError();
    }
    {
        std::lock_guard<std::mutex> lock(sc->ws_mutex);
        sc->ws_free.push_back(ws);
    }
    return rc;
}

// ---- pire_gpu_line_stream: a text from host memory as device frames of whole lines --------------------------------
//
// Slot k % 3 receives the line carried over from slot (k - 1) % 3 (device to device) and then the new bytes (host to
// device), all on the stream object's own stream.  The frame ends behind the last '\n' of the slot, found by a memrchr
// over the new bytes on the host (the carry has no newline by construction), and pire_gpu_split_lines cuts it on the
// device.  Before a slot is written, its stream waits for an event recorded on the caller's stream when the feed after
// the slot's frame began: the caller's work on that frame.  Nothing waits for the work on the frame just returned.

namespace pire_b200 {
namespace {

constexpr int kLineSlots = 3;
constexpr uint64_t kLineSlotDefault = 256ull << 20;    // tools/line_stream_bench.py, DESIGN.md 4
constexpr size_t kLinePad = 64;                // bytes behind a slot's text that vector loads may touch
constexpr size_t kStagePiece = 8u << 20;       // pageable input: staged and sent in pieces, so the two overlap

struct LineSlot {
    uint8_t* d_text = nullptr;
    size_t text_cap = 0;                       // bytes, kLinePad included
    uint64_t* d_off = nullptr;
    size_t off_cap = 0;                        // entries
    uint64_t used = 0;                         // carry + new bytes in the slot
    uint64_t framed = 0;                       // bytes of its frame; [framed, used) is carried to the next slot
    cudaEvent_t released = nullptr;            // the caller's work on this slot's frame
};

} // namespace
} // namespace pire_b200

struct pire_gpu_line_stream {
    int device = -1;
    uint64_t slot_bytes = 0;
    cudaStream_t copy = nullptr;
    cudaEvent_t ready = nullptr;
    pire_b200::LineSlot slot[pire_b200::kLineSlots];
    uint8_t* h_stage = nullptr;
    size_t stage_cap = 0;
    pire_b200::CopyPool* pool = nullptr;
    uint64_t frames = 0, first_line = 0, first_byte = 0;
    bool finished = false;

    ~pire_gpu_line_stream()
    {
        if (copy)
            cudaStreamSynchronize(copy);
        delete pool;
        cudaFreeHost(h_stage);
        for (pire_b200::LineSlot& s : slot) {
            cudaFree(s.d_text);
            cudaFree(s.d_off);
            if (s.released)
                cudaEventDestroy(s.released);
        }
        if (ready)
            cudaEventDestroy(ready);
        if (copy)
            cudaStreamDestroy(copy);
    }
};

namespace pire_b200 {
namespace {

int FeedLines(pire_gpu_line_stream* ls, const uint8_t* bytes, uint64_t n, bool last, cudaStream_t caller, uint64_t* consumed,
              pire_gpu_line_frame* frame)
{
    LineSlot& s = ls->slot[ls->frames % kLineSlots];
    LineSlot* prev = ls->frames ? &ls->slot[(ls->frames + kLineSlots - 1) % kLineSlots] : nullptr;
    // the work the caller has enqueued on the previous frame so far is what its slot waits for three frames on
    if (prev)
        CUDA_TRY(cudaEventRecord(prev->released, caller));
    const uint64_t carry = prev ? prev->used - prev->framed : 0;
    // room for the new bytes: a slot, or twice the carry once the carry fills half of one (a line longer than a slot)
    const uint64_t room = carry <= ls->slot_bytes / 2 ? ls->slot_bytes : 2 * carry;
    const uint64_t take = std::min<uint64_t>(n, room - carry);
    const uint64_t used = carry + take;

    // the slot's last frame (three feeds ago) may still be read by the caller's kernels
    CUDA_TRY(cudaStreamWaitEvent(ls->copy, s.released, 0));
    const size_t off_want = (size_t) (ls->slot_bytes / 64 + 2);
    if (s.text_cap < used + kLinePad || s.off_cap < off_want) {
        CUDA_TRY(cudaEventSynchronize(s.released));          // buffers are freed below, not only overwritten
        CUDA_TRY(GrowDevice(&s.d_text, &s.text_cap, (size_t) used + kLinePad));
        CUDA_TRY(GrowDevice(&s.d_off, &s.off_cap, off_want));
    }
    if (carry)
        CUDA_TRY(cudaMemcpyAsync(s.d_text, prev->d_text + prev->framed, carry, cudaMemcpyDeviceToDevice, ls->copy));
    if (take) {
        if (IsPinned(bytes)) {
            CUDA_TRY(cudaMemcpyAsync(s.d_text + carry, bytes, take, cudaMemcpyHostToDevice, ls->copy));
        } else {
            if (!ls->pool) {
                unsigned hw = std::thread::hardware_concurrency();
                size_t threads = EnvSize("PIRE_B200_HOST_THREADS", std::min<size_t>(8, std::max<unsigned>(1, hw / 4)));
                ls->pool = new CopyPool((unsigned) (threads > 1 ? threads - 1 : 0));
            }
            // the previous feed's copies from the staging buffer finished before it returned
            CUDA_TRY(GrowPinned(&ls->h_stage, &ls->stage_cap, (size_t) take));
            for (uint64_t at = 0; at < take; at += kStagePiece) {
                const size_t len = (size_t) std::min<uint64_t>(kStagePiece, take - at);
                ls->pool->Copy(ls->h_stage + at, bytes + at, len);
                CUDA_TRY(cudaMemcpyAsync(s.d_text + carry + at, ls->h_stage + at, len, cudaMemcpyHostToDevice, ls->copy));
            }
        }
    }
    // the frame: through the last newline of the slot, or everything once the text has ended
    const bool final = last && take == n;
    const void* nl = take ? memrchr(bytes, '\n', (size_t) take) : nullptr;
    const uint64_t framed = final ? used : nl ? carry + (uint64_t) (static_cast<const uint8_t*>(nl) - bytes) + 1 : 0;
    uint64_t lines = 0;
    if (framed) {
        for (;;) {
            int rc = pire_gpu_split_lines(s.d_text, framed, s.d_off, s.off_cap - 1, &lines, ls->device, ls->copy);
            if (rc == PIRE_GPU_OK)
                break;
            if (rc != PIRE_GPU_EINVAL || lines < s.off_cap)
                return rc;
            CUDA_TRY(GrowDevice(&s.d_off, &s.off_cap, (size_t) (lines + lines / 4 + 2)));   // the slot was released above
        }
    } else {
        CUDA_TRY(cudaMemsetAsync(s.d_off, 0, sizeof(uint64_t), ls->copy));
    }
    CUDA_TRY(cudaEventRecord(ls->ready, ls->copy));
    CUDA_TRY(cudaStreamWaitEvent(caller, ls->ready, 0));
    CUDA_TRY(cudaStreamSynchronize(ls->copy));                  // the caller's bytes are no longer referenced

    s.used = used;
    s.framed = framed;
    *frame = pire_gpu_line_frame{s.d_text, s.d_off, lines, framed, ls->first_line, ls->first_byte};
    *consumed = take;
    ls->first_line += lines;
    ls->first_byte += framed;
    ++ls->frames;
    ls->finished = final;
    return PIRE_GPU_OK;
}

} // namespace
} // namespace pire_b200

extern "C" int pire_gpu_line_stream_create(int device, uint64_t slot_bytes, pire_gpu_line_stream** out)
{
    if (!out)
        return Fail(PIRE_GPU_EINVAL, "out is null");
    *out = nullptr;
    if (device < 0)
        return Fail(PIRE_GPU_ENODEVICE, "a line stream needs a CUDA device");
    int count = 0;
    cudaError_t ce = cudaGetDeviceCount(&count);
    if (ce != cudaSuccess || device >= count) {
        (void) cudaGetLastError();
        return Fail(PIRE_GPU_ENODEVICE, ce != cudaSuccess ? std::string("no CUDA device: ") + cudaGetErrorString(ce)
                                                          : std::string("CUDA device index out of range"));
    }
    CUDA_TRY(cudaSetDevice(device));
    pire_gpu_line_stream* ls = new (std::nothrow) pire_gpu_line_stream;
    if (!ls)
        return Fail(PIRE_GPU_EINVAL, "out of memory");
    ls->device = device;
    ls->slot_bytes = slot_bytes ? slot_bytes : kLineSlotDefault;
    cudaError_t err = cudaStreamCreateWithFlags(&ls->copy, cudaStreamNonBlocking);
    if (err == cudaSuccess)
        err = cudaEventCreateWithFlags(&ls->ready, cudaEventDisableTiming);
    for (LineSlot& s : ls->slot)
        if (err == cudaSuccess)
            err = cudaEventCreateWithFlags(&s.released, cudaEventDisableTiming);
    if (err != cudaSuccess) {
        delete ls;
        return FailCuda(err, "pire_gpu_line_stream_create");
    }
    *out = ls;
    return PIRE_GPU_OK;
}

extern "C" int pire_gpu_line_stream_feed(pire_gpu_line_stream* ls, const uint8_t* bytes, uint64_t n, int last, void* stream,
                                         uint64_t* consumed, pire_gpu_line_frame* frame)
{
    if (!ls || !consumed || !frame || (!bytes && n))
        return Fail(PIRE_GPU_EINVAL, "null line stream, bytes, consumed or frame");
    *consumed = 0;
    if (ls->finished)
        return Fail(PIRE_GPU_EINVAL, "feed after the last piece of the text");
    CUDA_TRY(cudaSetDevice(ls->device));
    int rc;
    try {
        rc = FeedLines(ls, bytes, n, last != 0, static_cast<cudaStream_t>(stream), consumed, frame);
    } catch (const std::exception& e) {
        rc = Fail(PIRE_GPU_EINVAL, std::string("pire_gpu_line_stream_feed: ") + e.what());
    }
    if (rc != PIRE_GPU_OK) {
        *consumed = 0;
        cudaStreamSynchronize(ls->copy);           // nothing in flight still points at the caller's bytes
        (void) cudaGetLastError();
    }
    return rc;
}

extern "C" void pire_gpu_line_stream_destroy(pire_gpu_line_stream* ls)
{
    if (!ls)
        return;
    cudaSetDevice(ls->device);
    cudaDeviceSynchronize();                       // the caller's work on the last frames reads the slots
    delete ls;
}
