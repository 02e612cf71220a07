// batch_resume_check.cpp -- a batch of streams carried on round after round through include/pire_gpu.hpp's BatchRunner,
// from plain C++ (no Python).
//
//   batch_resume_check <scanner.pire> <n_strings> <len> <rounds> <seed>
//
// n pseudo-random strings of `len` bytes with planted literals are cut into `rounds` pieces each (len a multiple of
// 32 * rounds); every round is a fixed-length batch of the n pieces, laid out round-major.  The first round starts from
// Initialize() with Begin(), every later one from the states the previous one reached (Runner(gsc, From(d_state)),
// updated in place), the last one with End().  Match bits, accept masks and StateIndex must equal those of one
// pire_gpu_run_batch over the whole strings, and an untagged Runner must give pire_gpu_run_batch's words too.
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
    if (argc != 6) {
        std::fprintf(stderr, "usage: %s <scanner.pire> <n_strings> <len> <rounds> <seed>\n", argv[0]);
        return 2;
    }
    std::ifstream in(argv[1], std::ios::binary);
    std::vector<char> image((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
    const uint64_t n = std::strtoull(argv[2], nullptr, 10);
    const uint64_t len = std::strtoull(argv[3], nullptr, 10);
    const uint64_t rounds = std::strtoull(argv[4], nullptr, 10);
    uint64_t x = std::strtoull(argv[5], nullptr, 10) * 0x9E3779B97F4A7C15ull + 1;
    if (n == 0 || rounds == 0 || len % (32 * rounds) != 0) {
        std::fprintf(stderr, "len must be a multiple of 32 * rounds\n");
        return 2;
    }
    const uint64_t piece = len / rounds;
    std::vector<uint8_t> text(n * len);                 // string-major: string i at i * len
    const char* plants[] = {"error", "fatal", "https://", "GET ", "timeout"};
    for (uint64_t i = 0; i < text.size(); ++i) {
        x ^= x << 13, x ^= x >> 7, x ^= x << 17;
        text[i] = (uint8_t) (0x20 + (x >> 32) % 95);
    }
    for (uint64_t i = 0; i < n; i += 3) {               // across piece boundaries too
        const char* lit = plants[i % 5];
        const uint64_t at = (i * 7919) % (len - 8);
        std::memcpy(&text[i * len + at], lit, std::strlen(lit) < len - at ? std::strlen(lit) : len - at);
    }
    std::vector<uint8_t> by_round(n * len);             // round-major: piece r of string i at (r * n + i) * piece
    for (uint64_t r = 0; r < rounds; ++r)
        for (uint64_t i = 0; i < n; ++i)
            std::memcpy(&by_round[(r * n + i) * piece], &text[i * len + r * piece], piece);

    Scanner sc(image.data(), image.size(), 0);
    cudaStream_t stream;
    CU(cudaStreamCreate(&stream));
    uint8_t *d_text = nullptr, *d_rounds = nullptr;
    const uint64_t words = (n + 31) / 32;
    // [whole: bits, masks, states] [chained: bits, masks, states] [untagged runner: bits, masks, states]
    uint32_t* d_out = nullptr;
    const uint64_t stride = words + 2 * n;
    CU(cudaMalloc(&d_text, text.size()));
    CU(cudaMalloc(&d_rounds, by_round.size()));
    CU(cudaMalloc(&d_out, 3 * stride * 4));
    CU(cudaMemcpy(d_text, text.data(), text.size(), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_rounds, by_round.data(), by_round.size(), cudaMemcpyHostToDevice));
    CU(cudaMemset(d_out, 0xEE, 3 * stride * 4));
    uint32_t* whole = d_out;
    uint32_t* chained = d_out + stride;
    uint32_t* untagged = d_out + 2 * stride;

    Check(pire_gpu_run_batch(sc.Raw(), d_text, nullptr, len, n, PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END, whole, whole + words,
                             whole + words + n, stream), "pire_gpu_run_batch");
    Runner(sc).Begin().Run(Batch{d_text, nullptr, len, n}).End().Launch(untagged, untagged + words, untagged + words + n, stream);

    // round 0 from Initialize(); the state words are then carried on in place, with no synchronise in between
    uint32_t* d_state = chained + words + n;
    Runner(sc).Begin().Run(Batch{d_rounds, nullptr, piece, n}).Launch(nullptr, nullptr, d_state, stream);
    for (uint64_t r = 1; r < rounds; ++r) {
        BatchRunner next = Runner(sc, BatchRunner::From(d_state));
        next.Run(Batch{d_rounds + r * n * piece, nullptr, piece, n});
        if (r + 1 == rounds)
            next.End().Launch(chained, chained + words, d_state, stream);
        else
            next.Launch(nullptr, nullptr, d_state, stream);
    }
    std::vector<uint32_t> h(3 * stride);
    CU(cudaMemcpyAsync(h.data(), d_out, h.size() * 4, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    long mismatches = 0, finals = 0;
    for (uint64_t k = 0; k < stride; ++k) {
        if (rounds > 1 && h[stride + k] != h[k])
            ++mismatches;
        if (h[2 * stride + k] != h[k])
            ++mismatches;
    }
    for (uint64_t w = 0; w < words; ++w)
        finals += __builtin_popcount(h[w]);
    std::printf("%llu strings of %llu bytes in %llu rounds: %ld matches, %ld mismatches\n", (unsigned long long) n,
                (unsigned long long) len, (unsigned long long) rounds, finals, mismatches);
    cudaFree(d_text);
    cudaFree(d_rounds);
    cudaFree(d_out);
    cudaStreamDestroy(stream);
    return mismatches ? 1 : 0;
}
