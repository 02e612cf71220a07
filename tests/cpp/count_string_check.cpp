// count_string_check.cpp -- one long string counted through include/pire_gpu.hpp's StringCounter, from plain C++ (no
// Python): "how many times does each pattern occur in this file".
//
//   count_string_check <half_final_scanner.pire> <n_bytes> <seed>
//
// A pseudo-random string with planted literals is counted three ways: in one call, in pieces chained through one state
// word and one counts array (no synchronise in between), and by pire_gpu_count_batch as a CSR batch of one string; then
// the chain is resumed from the state its first half stopped in (Runner(sc, st)).  Counters, Final() and StateIndex
// must agree (the batch entry point gives counters and Final() only).
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
    uint64_t* d_counts = nullptr;      // [0] one call, [1] chained, [2] resumed: regs each
    uint32_t* d_batch = nullptr;       // count_batch's u32 row
    uint32_t* d_words = nullptr;       // [0..1] one call, [2..3] chained, [4..5] resumed, [6] batch match word
    uint64_t* d_off = nullptr;
    CU(cudaMalloc(&d_text, text.size()));
    CU(cudaMalloc(&d_counts, 3 * regs * 8));
    CU(cudaMalloc(&d_batch, regs * 4));
    CU(cudaMalloc(&d_words, 8 * 4));
    CU(cudaMalloc(&d_off, 16));
    CU(cudaMemcpy(d_text, text.data(), text.size(), cudaMemcpyHostToDevice));
    const uint8_t* s = d_text + 3;     // an odd start
    const uint64_t off[2] = {3, 3 + n};
    CU(cudaMemcpy(d_off, off, 16, cudaMemcpyHostToDevice));
    CU(cudaMemset(d_counts, 0, 3 * regs * 8));
    CU(cudaMemset(d_words, 0, 8 * 4));

    StringCounter(sc, d_counts, d_words + 1, d_words + 0, stream).Begin().Run(s, n).End();

    StringCounter chain(sc, d_counts + regs, d_words + 3, d_words + 2, stream);
    chain.Begin();
    const uint64_t cuts[] = {0, 1, 17, n / 3, n / 3, n / 2 + 5, n};
    for (int k = 0; k + 1 < (int) (sizeof(cuts) / sizeof(cuts[0])); ++k) {
        const uint64_t lo = cuts[k] < n ? cuts[k] : n, hi = cuts[k + 1] < n ? cuts[k + 1] : n;
        chain.Run(s + lo, hi - lo);
    }
    chain.End();

    // the first half without End(), then a fresh counter from the state it reached, in place, into the same counts
    StringCounter(sc, d_counts + 2 * regs, d_words + 5, d_words + 4, stream).Begin().Run(s, n / 2);
    StringCounter(sc, StringCounter::From(d_words + 5), d_counts + 2 * regs, d_words + 5, d_words + 4, stream).Run(s + n / 2, n - n / 2).End();

    Check(pire_gpu_count_batch(sc.Raw(), d_text, d_off, 0, 1, PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END, d_batch, d_words + 6, stream),
          "pire_gpu_count_batch");

    std::vector<uint64_t> c(3 * regs);
    std::vector<uint32_t> b(regs);
    uint32_t w[8];
    CU(cudaMemcpyAsync(c.data(), d_counts, c.size() * 8, cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(b.data(), d_batch, b.size() * 4, cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(w, d_words, sizeof(w), cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    long mismatches = 0;
    uint64_t total = 0;
    for (size_t r = 0; r < regs; ++r) {
        total += c[r];
        for (int k = 1; k < 3; ++k)
            if (c[k * regs + r] != c[r]) {
                std::printf("counter %zu, way %d: %llu, one call %llu\n", r, k, (unsigned long long) c[k * regs + r], (unsigned long long) c[r]);
                ++mismatches;
            }
        if (b[r] != c[r]) {
            std::printf("counter %zu: count_batch %u, one call %llu\n", r, b[r], (unsigned long long) c[r]);
            ++mismatches;
        }
    }
    for (int j : {2, 4})
        if (w[j] != w[0] || w[j + 1] != w[1]) {
            std::printf("words %d..%d: %08x %08x, one call %08x %08x\n", j, j + 1, w[j], w[j + 1], w[0], w[1]);
            ++mismatches;
        }
    if (w[6] != w[0]) {
        std::printf("count_batch final %u, one call %u\n", w[6], w[0]);
        ++mismatches;
    }
    std::printf("string of %llu bytes: %llu matches over %zu regexps, final %u state %u: %ld mismatches\n", (unsigned long long) n,
                (unsigned long long) total, regs, w[0], w[1], mismatches);
    cudaFree(d_text);
    cudaFree(d_counts);
    cudaFree(d_batch);
    cudaFree(d_words);
    cudaFree(d_off);
    cudaStreamDestroy(stream);
    return mismatches ? 1 : 0;
}
