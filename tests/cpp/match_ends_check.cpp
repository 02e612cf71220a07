// match_ends_check.cpp -- where the matches of one long string end, through include/pire_gpu.hpp's StringMatchEnds,
// from plain C++ (no Python): "regexp 3 occurs 41 times in this file: where?".
//
//   match_ends_check <half_final_scanner.pire> <n_bytes> <seed>
//
// A pseudo-random string with planted literals is counted by StringCounter, then its match ends are listed three ways:
// in one call, in pieces chained through one state word and one *d_found (no synchronise in between), and as a first
// half followed by a run resumed from the state it stopped in (Runner(sc, st)).  The three must write the same entries,
// their number must be the sum of the counters, the ends must ascend and the entries of regexp r must number Result(r).
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

int main(int argc, char** argv)
{
    using namespace Pire::Gpu;
    if (argc != 4) {
        std::fprintf(stderr, "usage: %s <scanner.pire> <n_bytes> <seed>\n", argv[0]);
        return 2;
    }
    std::ifstream in(argv[1], std::ios::binary);
    std::vector<char> image((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
    const uint64_t n = std::strtoull(argv[2], nullptr, 10);
    uint64_t x = std::strtoull(argv[3], nullptr, 10) * 0x9E3779B97F4A7C15ull + 1;
    std::vector<uint8_t> text(n + 3);
    const char* plants[] = {"error", "fatal", "https://", "GET ", "timeout"};
    for (uint64_t i = 0; i < text.size(); ++i) {
        x ^= x << 13, x ^= x >> 7, x ^= x << 17;
        text[i] = (uint8_t) (0x20 + (x >> 32) % 95);
    }
    for (uint64_t at = 777; at + 16 < n; at += 4099) {
        const char* lit = plants[(at / 4099) % 5];
        std::memcpy(&text[at], lit, std::strlen(lit));
    }

    Scanner sc(image.data(), image.size(), 0);
    const size_t regs = sc.RegexpsCount() ? sc.RegexpsCount() : 1;
    cudaStream_t stream;
    CU(cudaStreamCreate(&stream));
    uint8_t* d_text = nullptr;
    uint64_t* d_counts = nullptr;
    uint32_t* d_words = nullptr;       // [0..1] counter, [2..3] one call, [4..5] chained, [6..7] resumed
    uint64_t* d_found = nullptr;       // one call, chained, resumed
    CU(cudaMalloc(&d_text, text.size()));
    CU(cudaMalloc(&d_counts, regs * 8));
    CU(cudaMalloc(&d_words, 8 * 4));
    CU(cudaMalloc(&d_found, 3 * 8));
    CU(cudaMemcpy(d_text, text.data(), text.size(), cudaMemcpyHostToDevice));
    const uint8_t* s = d_text + 3;     // an odd start
    CU(cudaMemset(d_counts, 0, regs * 8));
    CU(cudaMemset(d_words, 0, 8 * 4));
    CU(cudaMemset(d_found, 0, 3 * 8));

    StringCounter(sc, d_counts, d_words + 1, d_words + 0, stream).Begin().Run(s, n).End();
    std::vector<uint64_t> counts(regs);
    CU(cudaMemcpyAsync(counts.data(), d_counts, regs * 8, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    uint64_t total = 0;
    for (uint64_t c : counts)
        total += c;

    const uint64_t cap = total ? total : 1;
    uint64_t* d_ends = nullptr;
    uint32_t* d_ids = nullptr;
    CU(cudaMalloc(&d_ends, 3 * cap * 8));
    CU(cudaMalloc(&d_ids, 3 * cap * 4));

    StringMatchEnds(sc, d_ends, d_ids, cap, d_found, d_words + 3, d_words + 2, stream).Begin().Run(s, n).End();

    StringMatchEnds chain(sc, d_ends + cap, d_ids + cap, cap, d_found + 1, d_words + 5, d_words + 4, stream);
    chain.Begin();
    const uint64_t cuts[] = {0, 1, 17, n / 3, n / 3, n / 2 + 5, n};
    for (int k = 0; k + 1 < (int) (sizeof(cuts) / sizeof(cuts[0])); ++k) {
        const uint64_t lo = cuts[k] < n ? cuts[k] : n, hi = cuts[k + 1] < n ? cuts[k + 1] : n;
        chain.Run(s + lo, hi - lo);
    }
    chain.End();

    // the first half without End(), then a fresh lister from the state it reached, in place, appending to the same
    // arrays: its ends count from its own first byte
    StringMatchEnds(sc, d_ends + 2 * cap, d_ids + 2 * cap, cap, d_found + 2, d_words + 7, d_words + 6, stream).Begin().Run(s, n / 2);
    CU(cudaStreamSynchronize(stream));
    uint64_t first_half = 0;
    CU(cudaMemcpy(&first_half, d_found + 2, 8, cudaMemcpyDeviceToHost));
    StringMatchEnds(sc, StringMatchEnds::From(d_words + 7), d_ends + 2 * cap, d_ids + 2 * cap, cap, d_found + 2, d_words + 7, d_words + 6,
                    stream).Run(s + n / 2, n - n / 2).End();

    std::vector<uint64_t> ends(3 * cap), found(3);
    std::vector<uint32_t> ids(3 * cap);
    uint32_t w[8];
    CU(cudaMemcpyAsync(ends.data(), d_ends, ends.size() * 8, cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(ids.data(), d_ids, ids.size() * 4, cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(found.data(), d_found, 3 * 8, cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(w, d_words, sizeof(w), cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    for (uint64_t k = first_half; k < total && k < cap; ++k)
        ends[2 * cap + k] += n / 2;

    long mismatches = 0;
    for (int j = 0; j < 3; ++j)
        if (found[j] != total) {
            std::printf("way %d: %llu entries, counters %llu\n", j, (unsigned long long) found[j], (unsigned long long) total);
            ++mismatches;
        }
    std::vector<uint64_t> hist(regs);
    for (uint64_t k = 0; k < total; ++k) {
        for (int j = 1; j < 3; ++j)
            if (ends[j * cap + k] != ends[k] || ids[j * cap + k] != ids[k]) {
                if (mismatches < 10)
                    std::printf("entry %llu, way %d: (%llu, %u), one call (%llu, %u)\n", (unsigned long long) k, j,
                                (unsigned long long) ends[j * cap + k], ids[j * cap + k], (unsigned long long) ends[k], ids[k]);
                ++mismatches;
            }
        if ((k && ends[k] < ends[k - 1]) || ends[k] > n || ids[k] >= regs) {
            std::printf("entry %llu: (%llu, %u) out of order or range\n", (unsigned long long) k, (unsigned long long) ends[k], ids[k]);
            ++mismatches;
        } else {
            ++hist[ids[k]];
        }
    }
    for (size_t r = 0; r < regs; ++r)
        if (hist[r] != counts[r]) {
            std::printf("regexp %zu: %llu entries, Result %llu\n", r, (unsigned long long) hist[r], (unsigned long long) counts[r]);
            ++mismatches;
        }
    for (int j : {2, 4, 6})
        if (w[j] != w[0] || w[j + 1] != w[1]) {
            std::printf("words %d..%d: %08x %08x, counter %08x %08x\n", j, j + 1, w[j], w[j + 1], w[0], w[1]);
            ++mismatches;
        }
    std::printf("string of %llu bytes: %llu match ends over %zu regexps, final %u state %u: %ld mismatches\n", (unsigned long long) n,
                (unsigned long long) total, regs, w[0], w[1], mismatches);
    cudaFree(d_text);
    cudaFree(d_counts);
    cudaFree(d_words);
    cudaFree(d_found);
    cudaFree(d_ends);
    cudaFree(d_ids);
    cudaStreamDestroy(stream);
    return mismatches ? 1 : 0;
}
