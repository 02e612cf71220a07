// string_check.cpp -- one long string through include/pire_gpu.hpp's StringRunner, from plain C++ (no Python): what
// a caller of tools/bench/bench.cpp's shape (Runner(sc).Begin().Run(begin, end).End() over a whole file) writes.
//
//   string_check <scanner.pire> <n_bytes> <seed>
//
// A pseudo-random string with planted literals is scanned three ways: in one call, in pieces chained through one
// device word (the state updated in place), and by pire_gpu_run_batch as a CSR batch of one string.  Match word,
// accept mask and StateIndex must agree; then the chain is resumed from the state it stopped in (Runner(sc, st)).
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
    for (uint64_t at = 777; at + 16 < n; at += 65537) {
        const char* lit = plants[(at / 65537) % 5];
        std::memcpy(&text[at], lit, std::strlen(lit));
    }

    Scanner sc(image.data(), image.size(), 0);
    cudaStream_t stream;
    CU(cudaStreamCreate(&stream));
    uint8_t* d_text = nullptr;
    // [0..2] one call, [4..6] chained, [8..10] batch, [12..14] resumed, [18] resumed through the three-argument form,
    // [20..22] through the five-argument form
    uint32_t* d_words = nullptr;
    uint64_t* d_off = nullptr;
    CU(cudaMalloc(&d_text, text.size()));
    CU(cudaMalloc(&d_words, 24 * 4));
    CU(cudaMalloc(&d_off, 16));
    CU(cudaMemcpy(d_text, text.data(), text.size(), cudaMemcpyHostToDevice));
    const uint8_t* s = d_text + 3;     // an odd start
    const uint64_t off[2] = {3, 3 + n};
    CU(cudaMemcpy(d_off, off, 16, cudaMemcpyHostToDevice));
    CU(cudaMemset(d_words, 0xEE, 24 * 4));

    StringRunner(sc, d_words + 2, d_words + 0, d_words + 1, stream).Begin().Run(s, n).End();

    StringRunner chain(sc, d_words + 6, d_words + 4, d_words + 5, stream);
    chain.Begin();
    const uint64_t cuts[] = {0, 1, 17, n / 3, n / 3, n / 2 + 5, n};
    for (int k = 0; k + 1 < (int) (sizeof(cuts) / sizeof(cuts[0])); ++k) {
        const uint64_t lo = cuts[k] < n ? cuts[k] : n, hi = cuts[k + 1] < n ? cuts[k + 1] : n;
        chain.Run(s + lo, hi - lo);
    }
    chain.End();

    Check(pire_gpu_run_batch(sc.Raw(), d_text, d_off, 0, 1, PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END, d_words + 8, d_words + 9,
                             d_words + 10, stream), "pire_gpu_run_batch");

    // Runner(sc, st): the first half without End(), then a fresh runner from the state it reached, in place
    CU(cudaMemset(d_words + 12, 0xEE, 3 * 4));
    StringRunner(sc, d_words + 14, d_words + 12, d_words + 13, stream).Begin().Run(s, n / 2);
    StringRunner(sc, StringRunner::From(d_words + 14), d_words + 14, d_words + 12, d_words + 13, stream).Run(s + n / 2, n - n / 2).End();

    // the same with the short forms, on the default stream: the start word tagged, the state word in place
    CU(cudaStreamSynchronize(stream));
    StringRunner(sc, d_words + 18).Begin().Run(s, n / 3);
    StringRunner(sc, StringRunner::From(d_words + 18), d_words + 18).Run(s + n / 3, n - n / 3).End();
    StringRunner(sc, d_words + 22).Begin().Run(s, n / 4);
    StringRunner(sc, StringRunner::From(d_words + 22), d_words + 22, d_words + 20, d_words + 21).Run(s + n / 4, n - n / 4).End();
    CU(cudaDeviceSynchronize());

    uint32_t w[24];
    CU(cudaMemcpyAsync(w, d_words, sizeof(w), cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    long mismatches = 0;
    for (int base : {4, 8, 12, 20})
        for (int j = 0; j < 3; ++j)
            if (w[base + j] != w[j]) {
                std::printf("word %d: %08x, one call %08x\n", base + j, w[base + j], w[j]);
                ++mismatches;
            }
    if (w[18] != w[2]) {
        std::printf("word 18: %08x, one call %08x\n", w[18], w[2]);
        ++mismatches;
    }
    for (int j : {16, 17, 19, 23})        // untouched: the short forms write no other word
        if (w[j] != 0xEEEEEEEEu) {
            std::printf("word %d written: %08x\n", j, w[j]);
            ++mismatches;
        }
    std::printf("string of %llu bytes: final %u mask %08x state %u: %ld mismatches\n", (unsigned long long) n, w[0], w[1], w[2],
                mismatches);
    cudaFree(d_text);
    cudaFree(d_words);
    cudaFree(d_off);
    cudaStreamDestroy(stream);
    return mismatches ? 1 : 0;
}
