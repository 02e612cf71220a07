// pair_check.cpp -- two scanners over one batch through include/pire_gpu.hpp's ScannerPair, from plain C++ (no Python).
//
//   pair_check <first.pire> <second.pire> <n_strings> <len> <rounds> <seed>
//
// n pseudo-random strings of `len` bytes with planted literals.  Runner(pair).Begin().Run(batch).End() must give each
// scanner the words of its own BatchRunner on the same batch.  The strings are also cut into `rounds` pieces (len a
// multiple of 32 * rounds), laid out round-major: Run(sc1, sc2, d_st1, d_st2, piece) carries both scanners' states on in
// place from Begin() (a first Runner(pair, From, From) round), and a last Runner(pair, From, From) round with End()
// must give the whole-string words again.
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
    if (argc != 7) {
        std::fprintf(stderr, "usage: %s <first.pire> <second.pire> <n_strings> <len> <rounds> <seed>\n", argv[0]);
        return 2;
    }
    const std::vector<char> image1 = ReadFile(argv[1]), image2 = ReadFile(argv[2]);
    const uint64_t n = std::strtoull(argv[3], nullptr, 10);
    const uint64_t len = std::strtoull(argv[4], nullptr, 10);
    const uint64_t rounds = std::strtoull(argv[5], nullptr, 10);
    uint64_t x = std::strtoull(argv[6], nullptr, 10) * 0x9E3779B97F4A7C15ull + 1;
    if (n == 0 || rounds == 0 || len % (32 * rounds) != 0) {
        std::fprintf(stderr, "len must be a multiple of 32 * rounds\n");
        return 2;
    }
    const uint64_t piece = len / rounds;
    std::vector<uint8_t> text(n * len);
    const char* plants[] = {"error", "fatal", "https://", "GET ", "hello  world"};
    for (uint64_t i = 0; i < text.size(); ++i) {
        x ^= x << 13, x ^= x >> 7, x ^= x << 17;
        text[i] = (uint8_t) (0x20 + (x >> 32) % 95);
    }
    for (uint64_t i = 0; i < n; i += 3) {
        const char* lit = plants[i % 5];
        const uint64_t at = i % 2 ? len - std::strlen(lit) : (i * 7919) % (len - 12);
        std::memcpy(&text[i * len + at], lit, std::strlen(lit) < len - at ? std::strlen(lit) : len - at);
    }
    std::vector<uint8_t> by_round(n * len);
    for (uint64_t r = 0; r < rounds; ++r)
        for (uint64_t i = 0; i < n; ++i)
            std::memcpy(&by_round[(r * n + i) * piece], &text[i * len + r * piece], piece);

    Scanner sc1(image1.data(), image1.size(), 0), sc2(image2.data(), image2.size(), 0);
    ScannerPair pair(sc1, sc2);
    cudaStream_t stream;
    CU(cudaStreamCreate(&stream));
    uint8_t *d_text = nullptr, *d_rounds = nullptr;
    const uint64_t words = (n + 31) / 32;
    const uint64_t stride = words + 2 * n;
    // per scanner: [single: bits, masks, states] [pair: ...] [chained: ...]
    uint32_t* d_out = nullptr;
    CU(cudaMalloc(&d_text, text.size()));
    CU(cudaMalloc(&d_rounds, by_round.size()));
    CU(cudaMalloc(&d_out, 6 * stride * 4));
    CU(cudaMemcpy(d_text, text.data(), text.size(), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_rounds, by_round.data(), by_round.size(), cudaMemcpyHostToDevice));
    CU(cudaMemset(d_out, 0xEE, 6 * stride * 4));
    auto out = [&](int scanner, int kind) {
        uint32_t* p = d_out + (uint64_t) (3 * scanner + kind) * stride;
        return RunOutputs{p, p + words, p + words + n};
    };
    const Batch whole{d_text, nullptr, len, n};
    const RunOutputs s1 = out(0, 0), s2 = out(1, 0);
    Runner(sc1).Begin().Run(whole).End().Launch(s1.MatchBits, s1.AcceptMasks, s1.StateIdx, stream);
    Runner(sc2).Begin().Run(whole).End().Launch(s2.MatchBits, s2.AcceptMasks, s2.StateIdx, stream);
    Runner(pair).Begin().Run(whole).End().Launch(out(0, 1), out(1, 1), stream);

    // chained: round 0 with Begin() from Initialize(), the middle rounds through Run(sc1, sc2, ...), the last with End()
    uint32_t* st1 = out(0, 2).StateIdx;
    uint32_t* st2 = out(1, 2).StateIdx;
    Runner(pair).Begin().Run(Batch{d_rounds, nullptr, piece, n}).Launch({nullptr, nullptr, st1}, {nullptr, nullptr, st2}, stream);
    for (uint64_t r = 1; r + 1 < rounds; ++r)
        Run(sc1, sc2, st1, st2, Batch{d_rounds + r * n * piece, nullptr, piece, n}, stream);
    if (rounds > 1)
        Runner(pair, BatchRunner::From(st1), BatchRunner::From(st2))
            .Run(Batch{d_rounds + (rounds - 1) * n * piece, nullptr, piece, n})
            .End()
            .Launch(out(0, 2), out(1, 2), stream);

    std::vector<uint32_t> h(6 * stride);
    CU(cudaMemcpyAsync(h.data(), d_out, h.size() * 4, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    long mismatches = 0, finals1 = 0, finals2 = 0;
    for (int s = 0; s < 2; ++s)
        for (uint64_t k = 0; k < stride; ++k) {
            const uint32_t want = h[(3 * s) * stride + k];
            if (h[(3 * s + 1) * stride + k] != want)
                ++mismatches;
            if (rounds > 1 && h[(3 * s + 2) * stride + k] != want)
                ++mismatches;
        }
    for (uint64_t w = 0; w < words; ++w) {
        finals1 += __builtin_popcount(h[w]);
        finals2 += __builtin_popcount(h[3 * stride + w]);
    }
    std::printf("%llu strings of %llu bytes in %llu rounds: %ld + %ld matches, %ld mismatches\n", (unsigned long long) n,
                (unsigned long long) len, (unsigned long long) rounds, finals1, finals2, mismatches);
    cudaFree(d_text);
    cudaFree(d_rounds);
    cudaFree(d_out);
    cudaStreamDestroy(stream);
    return mismatches ? 1 : 0;
}
