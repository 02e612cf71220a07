// batch_count_check.cpp -- many streams counted through include/pire_gpu.hpp's BatchCounter, from plain C++ (no Python):
// "how many times does each pattern occur in each of these connections".
//
//   batch_count_check <half_final_scanner.pire> <n> <length> <rounds> <seed>
//
// n pseudo-random strings of `length` bytes with planted literals are counted three ways: by pire_gpu_count_batch over
// the whole strings; by one BatchCounter fed `rounds` pieces of every string, chained through one state array and one
// counts array (no synchronise in between); and by a BatchCounter that stops after the first half of the rounds and a
// second one resumed from the states it reached (BatchCounter::From, in place).  Counters and Final() must agree, and
// the states must equal pire_gpu_run_batch's over the whole strings.
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
        std::fprintf(stderr, "usage: %s <scanner.pire> <n> <length> <rounds> <seed>\n", argv[0]);
        return 2;
    }
    std::ifstream in(argv[1], std::ios::binary);
    std::vector<char> image((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
    const uint64_t n = std::strtoull(argv[2], nullptr, 10);
    const uint64_t length = std::strtoull(argv[3], nullptr, 10);
    const int rounds = std::atoi(argv[4]);
    if (rounds < 2) {
        std::fprintf(stderr, "rounds must be at least 2: the resumed counter takes over after rounds / 2\n");
        return 2;
    }
    uint64_t x = std::strtoull(argv[5], nullptr, 10) * 0x9E3779B97F4A7C15ull + 1;
    std::vector<uint8_t> text(n * length);
    const char* plants[] = {"error", "fatal", "https://", "GET ", "timeout"};
    for (uint64_t i = 0; i < text.size(); ++i) {
        x ^= x << 13, x ^= x >> 7, x ^= x << 17;
        text[i] = (uint8_t) (0x20 + (x >> 32) % 95);
    }
    for (uint64_t i = 0; i < n && length >= 16; i += 3) {
        const char* lit = plants[i % 5];
        std::memcpy(&text[i * length + (i * 7) % (length - 8)], lit, std::strlen(lit));
    }

    Scanner sc(image.data(), image.size(), 0);
    const size_t regs = sc.RegexpsCount() ? sc.RegexpsCount() : 1;
    const uint64_t words = (n + 31) / 32;
    cudaStream_t stream;
    CU(cudaStreamCreate(&stream));
    uint8_t* d_text = nullptr;          // the whole strings, then round r's pieces at d_pieces[r]
    std::vector<uint8_t*> d_pieces(rounds, nullptr);
    uint32_t* d_batch = nullptr;        // count_batch's u32 rows
    uint64_t* d_counts = nullptr;       // [0] chained, [1] resumed: n * regs each
    uint32_t* d_state = nullptr;        // [0] chained, [1] resumed, [2] run_batch: n each
    uint32_t* d_bits = nullptr;         // [0] count_batch, [1] chained, [2] resumed, [3] run_batch: words each
    CU(cudaMalloc(&d_text, text.size() + 1));
    CU(cudaMalloc(&d_batch, n * regs * 4 + 4));
    CU(cudaMalloc(&d_counts, 2 * n * regs * 8 + 8));
    CU(cudaMalloc(&d_state, 3 * n * 4 + 4));
    CU(cudaMalloc(&d_bits, 4 * words * 4 + 4));
    CU(cudaMemcpy(d_text, text.data(), text.size(), cudaMemcpyHostToDevice));
    CU(cudaMemset(d_counts, 0, 2 * n * regs * 8));
    CU(cudaMemset(d_bits, 0, 4 * words * 4));
    std::vector<uint64_t> cut(rounds + 1);
    for (int r = 0; r <= rounds; ++r)
        cut[r] = length * r / rounds;
    for (int r = 0; r < rounds; ++r) {
        const uint64_t len = cut[r + 1] - cut[r];
        std::vector<uint8_t> piece(n * len);
        for (uint64_t i = 0; i < n; ++i)
            std::memcpy(&piece[i * len], &text[i * length + cut[r]], len);
        CU(cudaMalloc(&d_pieces[r], piece.size() + 1));
        CU(cudaMemcpy(d_pieces[r], piece.data(), piece.size(), cudaMemcpyHostToDevice));
    }
    auto piece = [&](int r) { return Batch{d_pieces[r], nullptr, cut[r + 1] - cut[r], n}; };
    const unsigned both = PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END;

    Check(pire_gpu_count_batch(sc.Raw(), d_text, nullptr, length, n, both, d_batch, d_bits, stream), "pire_gpu_count_batch");
    Runner(sc).Begin().Run(Batch{d_text, nullptr, length, n}).End().Launch(d_bits + 3 * words, nullptr, d_state + 2 * n, stream);

    BatchCounter chain(sc, n, d_counts, d_state, d_bits + words, stream);
    chain.Begin();
    for (int r = 0; r < rounds; ++r)
        chain.Run(piece(r));
    chain.End();

    uint64_t* c1 = d_counts + n * regs;
    uint32_t* s1 = d_state + n;
    BatchCounter first(sc, n, c1, s1, nullptr, stream);
    first.Begin();
    for (int r = 0; r < rounds / 2; ++r)
        first.Run(piece(r));
    BatchCounter rest(sc, BatchCounter::From(s1), n, c1, s1, d_bits + 2 * words, stream);
    for (int r = rounds / 2; r < rounds; ++r)
        rest.Run(piece(r));
    rest.End();

    std::vector<uint32_t> batch(n * regs), state(3 * n), bits(4 * words);
    std::vector<uint64_t> counts(2 * n * regs);
    CU(cudaMemcpyAsync(batch.data(), d_batch, batch.size() * 4, cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(counts.data(), d_counts, counts.size() * 8, cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(state.data(), d_state, state.size() * 4, cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(bits.data(), d_bits, bits.size() * 4, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    long mismatches = 0;
    uint64_t total = 0;
    for (uint64_t k = 0; k < n * regs; ++k) {
        total += batch[k];
        for (int way = 0; way < 2; ++way)
            if (counts[way * n * regs + k] != batch[k] && mismatches++ < 10)
                std::printf("string %llu counter %llu, way %d: %llu, count_batch %u\n", (unsigned long long) (k / regs),
                            (unsigned long long) (k % regs), way, (unsigned long long) counts[way * n * regs + k], batch[k]);
    }
    for (uint64_t i = 0; i < n; ++i)
        for (int way = 0; way < 2; ++way)
            if (state[way * n + i] != state[2 * n + i] && mismatches++ < 10)
                std::printf("string %llu, way %d: state %u, run_batch %u\n", (unsigned long long) i, way, state[way * n + i], state[2 * n + i]);
    for (uint64_t w = 0; w < words; ++w)
        for (int way = 1; way < 4; ++way)
            if (bits[way * words + w] != bits[w] && mismatches++ < 10)
                std::printf("bitmap word %llu, way %d: %08x, count_batch %08x\n", (unsigned long long) w, way, bits[way * words + w], bits[w]);
    std::printf("%llu strings of %llu bytes in %d rounds: %llu matches over %zu regexps: %ld mismatches\n", (unsigned long long) n,
                (unsigned long long) length, rounds, (unsigned long long) total, regs, mismatches);
    cudaFree(d_text);
    for (uint8_t* p : d_pieces)
        cudaFree(p);
    cudaFree(d_batch);
    cudaFree(d_counts);
    cudaFree(d_state);
    cudaFree(d_bits);
    cudaStreamDestroy(stream);
    return mismatches ? 1 : 0;
}
