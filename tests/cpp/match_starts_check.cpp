// match_starts_check.cpp -- where the matches of one long string start, through include/pire_gpu.hpp's StringMatchEnds
// and MatchStarts, from plain C++ (no Python): ends plus starts over a text that arrives in pieces.
//
//   match_starts_check <half_final_scanner.pire> <reversed_scanner.pire> <n_bytes> <seed>
//
// A pseudo-random string with planted literals gets its match ends and starts in one call each.  Then the same text is
// fed in pieces: before each piece the running *d_found is copied into d_first (8 bytes, device to device), the ends of
// the piece are appended, and the starts of the new entries are found in a window of the piece plus the 4 KiB before it
// (the last piece after End(), with END).  Entries whose walk stayed inside the window (open == 0) must have the one
// call's start; the open ones are found again in the window from the text's start, and must then have it too.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <vector>

#include "pire_gpu.hpp"

#define CU(expr)                                                                          \
    do {                                                                                  \
        cudaError_t e__ = (expr);                                                         \
        if (e__ != cudaSuccess) {                                                         \
            std::fprintf(stderr, "%s: %s\n", #expr, cudaGetErrorString(e__));             \
            std::exit(2);                                                                 \
        }                                                                                 \
    } while (0)

static std::vector<char> ReadFile(const char* path)
{
    std::ifstream in(path, std::ios::binary);
    return std::vector<char>((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
}

int main(int argc, char** argv)
{
    using namespace Pire::Gpu;
    if (argc != 5) {
        std::fprintf(stderr, "usage: %s <half_final.pire> <reversed.pire> <n_bytes> <seed>\n", argv[0]);
        return 2;
    }
    const std::vector<char> fwd_image = ReadFile(argv[1]), rev_image = ReadFile(argv[2]);
    const uint64_t n = std::strtoull(argv[3], nullptr, 10);
    uint64_t x = std::strtoull(argv[4], nullptr, 10) * 0x9E3779B97F4A7C15ull + 1;
    std::vector<uint8_t> text(n + 1);
    const char* plants[] = {"error", "fatal", "https://", "GET ", "timeout", "hello  world", "ABCDEFGHIJKLMNOPQRSTUVWXYZ"};
    for (uint64_t i = 0; i < text.size(); ++i) {
        x ^= x << 13, x ^= x >> 7, x ^= x << 17;
        text[i] = (uint8_t) (0x20 + (x >> 32) % 95);
    }
    for (uint64_t at = 501; at + 32 < n; at += 2053) {
        const char* lit = plants[(at / 2053) % 7];
        std::memcpy(&text[at], lit, std::strlen(lit));
    }

    Scanner fwd(fwd_image.data(), fwd_image.size(), 0), rev(rev_image.data(), rev_image.size(), 0);
    cudaStream_t stream;
    CU(cudaStreamCreate(&stream));
    const uint64_t cap = 4 * n + 16;
    uint8_t* d_text = nullptr;
    uint64_t *d_ends = nullptr, *d_starts = nullptr, *d_words = nullptr;     // words: found one call, found chained, first
    uint32_t *d_ids = nullptr, *d_state = nullptr;
    uint8_t* d_open = nullptr;
    CU(cudaMalloc(&d_text, n + 1));
    CU(cudaMalloc(&d_ends, 2 * cap * 8));
    CU(cudaMalloc(&d_ids, 2 * cap * 4));
    CU(cudaMalloc(&d_starts, 2 * cap * 8));
    CU(cudaMalloc(&d_open, 2 * cap));
    CU(cudaMalloc(&d_words, 3 * 8));
    CU(cudaMalloc(&d_state, 4 * 4));
    CU(cudaMemcpy(d_text, text.data(), n + 1, cudaMemcpyHostToDevice));
    CU(cudaMemset(d_words, 0, 3 * 8));

    StringMatchEnds one(fwd, d_ends, d_ids, cap, d_words, d_state, d_state + 1, stream);
    one.Begin().Run(d_text, n).End();
    MatchStarts(rev, one, d_text, n, 0, d_starts, d_open);

    const uint64_t back = 4096;
    StringMatchEnds chain(fwd, d_ends + cap, d_ids + cap, cap, d_words + 1, d_state + 2, d_state + 3, stream);
    chain.Begin();
    const uint64_t cuts[] = {0, 1, n / 5, n / 3, n / 2 + 7, n};
    const int pieces = (int) (sizeof(cuts) / sizeof(cuts[0])) - 1;
    for (int k = 0; k < pieces; ++k) {
        const uint64_t lo = cuts[k] < n ? cuts[k] : n;
        uint64_t hi = cuts[k + 1] < n ? cuts[k + 1] : n;
        if (hi < lo)                                                    // a short text: the piece is empty
            hi = lo;
        const uint64_t wlo = lo > back ? lo - back : 0;
        CU(cudaMemcpyAsync(d_words + 2, d_words + 1, 8, cudaMemcpyDeviceToDevice, stream));
        chain.Run(d_text + lo, hi - lo);
        const bool last = k + 1 == pieces;
        if (last)
            chain.End();
        MatchStarts(rev, chain, d_text + wlo, hi - wlo, wlo, d_starts + cap, d_open + cap, wlo == 0, last, 0, d_words + 2);
    }
    std::vector<uint64_t> ends(2 * cap), starts(2 * cap), words(3);
    std::vector<uint32_t> ids(2 * cap);
    std::vector<uint8_t> open(2 * cap);
    CU(cudaMemcpyAsync(words.data(), d_words, 3 * 8, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    const uint64_t total = words[0];
    long mismatches = 0, reopened = 0;
    if (words[1] != total || total > cap) {
        std::printf("%llu entries chained, %llu in one call (capacity %llu)\n", (unsigned long long) words[1],
                    (unsigned long long) total, (unsigned long long) cap);
        ++mismatches;
    }
    // the open entries once more, in the window from the text's start up to their own end
    CU(cudaMemcpyAsync(open.data(), d_open, 2 * cap, cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(ends.data(), d_ends, 2 * cap * 8, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    for (uint64_t k = 0; k < total && !mismatches; ++k)
        if (open[cap + k]) {
            const uint64_t e = ends[cap + k];
            CU(cudaMemcpyAsync(d_words + 2, &k, 8, cudaMemcpyHostToDevice, stream));
            const uint64_t stop = k + 1;
            uint64_t* d_stop = d_words + 1;                       // the chain's count, lowered to this one entry
            CU(cudaMemcpyAsync(d_stop, &stop, 8, cudaMemcpyHostToDevice, stream));
            MatchStarts(rev, chain, d_text, e, 0, d_starts + cap, d_open + cap, true, e == n, 0, d_words + 2);
            CU(cudaStreamSynchronize(stream));
            ++reopened;
        }
    CU(cudaMemcpyAsync(starts.data(), d_starts, 2 * cap * 8, cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(ids.data(), d_ids, 2 * cap * 4, cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(open.data(), d_open, 2 * cap, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    uint64_t with_start = 0;
    for (uint64_t k = 0; k < total && k < cap; ++k) {
        if (ends[cap + k] != ends[k] || ids[cap + k] != ids[k] || starts[cap + k] != starts[k] || open[k]) {
            if (mismatches < 10)
                std::printf("entry %llu: chained (%llu, %llu, %u), one call (%llu, %llu, %u) open %u\n", (unsigned long long) k,
                            (unsigned long long) starts[cap + k], (unsigned long long) ends[cap + k], ids[cap + k],
                            (unsigned long long) starts[k], (unsigned long long) ends[k], ids[k], open[k]);
            ++mismatches;
        }
        if (starts[k] != PIRE_GPU_NO_START) {
            ++with_start;
            if (starts[k] > ends[k])
                ++mismatches;
        }
    }
    std::printf("string of %llu bytes: %llu match ends, %llu with a start, %ld found again in a wider window: %ld mismatches\n",
                (unsigned long long) n, (unsigned long long) total, (unsigned long long) with_start, reopened, mismatches);
    cudaFree(d_text);
    cudaFree(d_ends);
    cudaFree(d_ids);
    cudaFree(d_starts);
    cudaFree(d_open);
    cudaFree(d_words);
    cudaFree(d_state);
    cudaStreamDestroy(stream);
    return mismatches ? 1 : 0;
}
