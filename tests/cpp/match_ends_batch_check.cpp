// match_ends_batch_check.cpp -- where the matches of many streams end, through include/pire_gpu.hpp's BatchMatchEnds,
// from plain C++ (no Python): "regexp 3 occurred 41 times in connection 17: where?".
//
//   match_ends_batch_check <half_final_scanner.pire> <n> <length> <rounds> <seed>
//
// n pseudo-random strings of `length` bytes with planted literals go through three front ends: one BatchMatchEnds call
// over the whole strings; a BatchMatchEnds fed `rounds` pieces of every string, chained through one state array and
// one position array, resumed half way with BatchMatchEnds::From (no synchronise in between); and a BatchCounter fed the
// same pieces.  The chained entries, taken stream by stream, must equal the whole-string call's entries byte for byte,
// every stream's per-id histogram must equal its BatchCounter row, and states and Final() must agree.
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

struct Entries {
    uint64_t found = 0;
    std::vector<uint32_t> strings, ids;
    std::vector<uint64_t> ends;
};

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
        std::fprintf(stderr, "rounds must be at least 2: the resumed front end takes over after rounds / 2\n");
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
    uint8_t* d_text = nullptr;
    std::vector<uint8_t*> d_pieces(rounds, nullptr);
    std::vector<uint64_t> cut(rounds + 1);
    for (int r = 0; r <= rounds; ++r)
        cut[r] = length * r / rounds;
    CU(cudaMalloc(&d_text, text.size() + 1));
    CU(cudaMemcpy(d_text, text.data(), text.size(), cudaMemcpyHostToDevice));
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

    // the total, from BatchCounter over the pieces
    uint64_t* d_counts = nullptr;
    uint32_t* d_state = nullptr;        // [0] counter, [1] whole, [2] chained: n each
    uint32_t* d_bits = nullptr;         // [0] counter, [1] whole, [2] chained: words each
    uint64_t* d_pos = nullptr;          // [0] whole, [1] chained: n each
    uint64_t* d_found = nullptr;        // [0] whole, [1] chained
    CU(cudaMalloc(&d_counts, n * regs * 8 + 8));
    CU(cudaMalloc(&d_state, 3 * n * 4 + 4));
    CU(cudaMalloc(&d_bits, 3 * words * 4 + 4));
    CU(cudaMalloc(&d_pos, 2 * n * 8 + 8));
    CU(cudaMalloc(&d_found, 2 * 8));
    CU(cudaMemset(d_counts, 0, n * regs * 8));
    CU(cudaMemset(d_pos, 0, 2 * n * 8));
    CU(cudaMemset(d_found, 0, 2 * 8));
    BatchCounter counter(sc, n, d_counts, d_state, d_bits, stream);
    counter.Begin();
    for (int r = 0; r < rounds; ++r)
        counter.Run(piece(r));
    counter.End();
    std::vector<uint64_t> counts(n * regs);
    CU(cudaMemcpyAsync(counts.data(), d_counts, counts.size() * 8, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    uint64_t total = 0;
    for (uint64_t c : counts)
        total += c;

    const uint64_t cap = total + 1;
    uint32_t *d_strings = nullptr, *d_ids = nullptr;
    uint64_t* d_ends = nullptr;
    CU(cudaMalloc(&d_strings, 2 * cap * 4));
    CU(cudaMalloc(&d_ids, 2 * cap * 4));
    CU(cudaMalloc(&d_ends, 2 * cap * 8));

    BatchMatchEnds whole(sc, n, d_pos, d_strings, d_ends, d_ids, cap, d_found, d_state + n, d_bits + words, stream);
    whole.Begin().Run(Batch{d_text, nullptr, length, n}).End();

    uint32_t* s2 = d_state + 2 * n;
    BatchMatchEnds first(sc, n, d_pos + n, d_strings + cap, d_ends + cap, d_ids + cap, cap, d_found + 1, s2, nullptr, stream);
    first.Begin();
    for (int r = 0; r < rounds / 2; ++r)
        first.Run(piece(r));
    BatchMatchEnds rest(sc, BatchMatchEnds::From(s2), n, d_pos + n, d_strings + cap, d_ends + cap, d_ids + cap, cap, d_found + 1, s2,
                        d_bits + 2 * words, stream);
    for (int r = rounds / 2; r < rounds; ++r)
        rest.Run(piece(r));
    rest.End();

    Entries e[2];
    std::vector<uint32_t> state(3 * n), bits(3 * words);
    std::vector<uint64_t> pos(2 * n);
    for (int way = 0; way < 2; ++way) {
        e[way].strings.resize(cap);
        e[way].ids.resize(cap);
        e[way].ends.resize(cap);
        CU(cudaMemcpyAsync(&e[way].found, d_found + way, 8, cudaMemcpyDeviceToHost, stream));
        CU(cudaMemcpyAsync(e[way].strings.data(), d_strings + way * cap, cap * 4, cudaMemcpyDeviceToHost, stream));
        CU(cudaMemcpyAsync(e[way].ids.data(), d_ids + way * cap, cap * 4, cudaMemcpyDeviceToHost, stream));
        CU(cudaMemcpyAsync(e[way].ends.data(), d_ends + way * cap, cap * 8, cudaMemcpyDeviceToHost, stream));
    }
    CU(cudaMemcpyAsync(state.data(), d_state, state.size() * 4, cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(bits.data(), d_bits, bits.size() * 4, cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(pos.data(), d_pos, pos.size() * 8, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));

    long mismatches = 0;
    for (int way = 0; way < 2; ++way)
        if (e[way].found != total && mismatches++ < 10)
            std::printf("way %d: %llu entries, BatchCounter %llu\n", way, (unsigned long long) e[way].found, (unsigned long long) total);
    // the whole-string call: ordered by stream, its histograms the counter's rows
    std::vector<uint64_t> hist(n * regs, 0);
    std::vector<uint64_t> first_of(n + 1, 0);           // the whole call's first entry of every stream
    for (uint64_t k = 0; k < total && k < cap; ++k) {
        const uint32_t i = e[0].strings[k];
        if ((i >= n || (k && i < e[0].strings[k - 1]) || e[0].ids[k] >= regs || e[0].ends[k] > length) && mismatches++ < 10) {
            std::printf("whole call, entry %llu: (%u, %llu, %u) out of order or range\n", (unsigned long long) k, i,
                        (unsigned long long) e[0].ends[k], e[0].ids[k]);
            continue;
        }
        if (i < n && e[0].ids[k] < regs)
            ++hist[i * regs + e[0].ids[k]], ++first_of[i + 1];
    }
    for (uint64_t i = 0; i < n; ++i)
        first_of[i + 1] += first_of[i];
    for (uint64_t k = 0; k < n * regs; ++k)
        if (hist[k] != counts[k] && mismatches++ < 10)
            std::printf("stream %llu regexp %llu: %llu entries, BatchCounter %llu\n", (unsigned long long) (k / regs),
                        (unsigned long long) (k % regs), (unsigned long long) hist[k], (unsigned long long) counts[k]);
    // the chained entries, stream by stream, are the whole call's
    std::vector<uint64_t> next(first_of.begin(), first_of.end() - 1);
    for (uint64_t k = 0; k < total && k < cap; ++k) {
        const uint32_t i = e[1].strings[k];
        if (i >= n) {
            if (mismatches++ < 10)
                std::printf("chained entry %llu: stream %u\n", (unsigned long long) k, i);
            continue;
        }
        const uint64_t at = next[i]++;
        if ((at >= first_of[i + 1] || e[1].ends[k] != e[0].ends[at] || e[1].ids[k] != e[0].ids[at]) && mismatches++ < 10)
            std::printf("stream %u: chained entry %llu differs from the whole call's\n", i, (unsigned long long) k);
    }
    for (uint64_t i = 0; i < n; ++i) {
        for (int way = 1; way < 3; ++way)
            if (state[way * n + i] != state[i] && mismatches++ < 10)
                std::printf("stream %llu, way %d: state %u, BatchCounter %u\n", (unsigned long long) i, way, state[way * n + i], state[i]);
        for (int way = 0; way < 2; ++way)
            if (pos[way * n + i] != length && mismatches++ < 10)
                std::printf("stream %llu, way %d: position %llu\n", (unsigned long long) i, way, (unsigned long long) pos[way * n + i]);
    }
    for (uint64_t w = 0; w < words; ++w)
        for (int way = 1; way < 3; ++way)
            if (bits[way * words + w] != bits[w] && mismatches++ < 10)
                std::printf("bitmap word %llu, way %d: %08x, BatchCounter %08x\n", (unsigned long long) w, way, bits[way * words + w], bits[w]);
    std::printf("%llu streams of %llu bytes in %d rounds: %llu entries over %zu regexps: %ld mismatches\n", (unsigned long long) n,
                (unsigned long long) length, rounds, (unsigned long long) total, regs, mismatches);
    cudaFree(d_text);
    for (uint8_t* p : d_pieces)
        cudaFree(p);
    cudaFree(d_counts);
    cudaFree(d_state);
    cudaFree(d_bits);
    cudaFree(d_pos);
    cudaFree(d_found);
    cudaFree(d_strings);
    cudaFree(d_ids);
    cudaFree(d_ends);
    cudaStreamDestroy(stream);
    return mismatches ? 1 : 0;
}
