// match_ends_lines_check.cpp -- where the matches end and start in every line of a text, through include/pire_gpu.hpp's
// LineMatchEnds and MatchStarts, from plain C++ (no Python).
//
//   match_ends_lines_check <half_final_scanner.pire> <reversed_scanner.pire> <n_lines> <seed>
//
// A pseudo-random text of lines (some empty, some with planted literals, \r\n on some, no final newline) is split on the
// device (pire_gpu_split_lines) and gets its ends and starts in one call each.  Every line is then run alone through
// StringMatchEnds (the line's bytes, base = its offset) and MatchStarts' string form with the line as its window; the
// entries and starts must be the same, in the same order.  Prints "<n> entries: <m> mismatches".
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

template <class T>
static std::vector<T> Host(const T* d, uint64_t n)
{
    std::vector<T> h(n);
    if (n)
        CU(cudaMemcpy(h.data(), d, n * sizeof(T), cudaMemcpyDeviceToHost));
    return h;
}

int main(int argc, char** argv)
{
    using namespace Pire::Gpu;
    if (argc != 5) {
        std::fprintf(stderr, "usage: %s <half_final.pire> <reversed.pire> <n_lines> <seed>\n", argv[0]);
        return 2;
    }
    const std::vector<char> fwd_image = ReadFile(argv[1]), rev_image = ReadFile(argv[2]);
    const uint64_t want_lines = std::strtoull(argv[3], nullptr, 10);
    uint64_t x = std::strtoull(argv[4], nullptr, 10) * 0x9E3779B97F4A7C15ull + 1;
    auto next = [&x] { x ^= x << 13, x ^= x >> 7, x ^= x << 17; return x >> 32; };
    const char* plants[] = {"error", "fatal", "https://", "GET ", "timeout", "hello  world"};
    std::vector<uint8_t> text;
    for (uint64_t l = 0; l < want_lines; ++l) {
        if (l)
            text.push_back('\n');
        const uint64_t len = next() % 7 == 0 ? 0 : next() % 140;
        const size_t at = text.size();
        for (uint64_t k = 0; k < len; ++k)
            text.push_back((uint8_t) (0x20 + next() % 95));
        const char* lit = plants[next() % 6];
        if (len > 20 && next() % 2)
            std::memcpy(&text[at + next() % (len - 13)], lit, std::strlen(lit));
        if (len && next() % 5 == 0)
            text.push_back('\r');
    }

    Scanner fwd(fwd_image.data(), fwd_image.size(), 0), rev(rev_image.data(), rev_image.size(), 0);
    uint8_t* d_text = nullptr;
    uint64_t* d_offs = nullptr;
    CU(cudaMalloc(&d_text, text.size() + 1));
    CU(cudaMalloc(&d_offs, (want_lines + 2) * 8));
    if (!text.empty())
        CU(cudaMemcpy(d_text, text.data(), text.size(), cudaMemcpyHostToDevice));
    uint64_t n_lines = 0;
    Check(pire_gpu_split_lines(d_text, text.size(), d_offs, want_lines + 1, &n_lines, 0, nullptr), "pire_gpu_split_lines");
    const std::vector<uint64_t> offs = Host(d_offs, n_lines + 1);
    const Batch lines = {d_text, d_offs, 0, n_lines};

    const uint64_t cap = 16 * text.size() + 64;
    uint32_t *d_lines = nullptr, *d_ids = nullptr, *d_ids1 = nullptr, *d_state = nullptr;
    uint64_t *d_ends = nullptr, *d_found = nullptr, *d_starts = nullptr, *d_ends1 = nullptr, *d_found1 = nullptr, *d_starts1 = nullptr;
    CU(cudaMalloc(&d_lines, cap * 4));
    CU(cudaMalloc(&d_ids, cap * 4));
    CU(cudaMalloc(&d_ends, cap * 8));
    CU(cudaMalloc(&d_starts, cap * 8));
    CU(cudaMalloc(&d_ids1, 4096 * 4));
    CU(cudaMalloc(&d_ends1, 4096 * 8));
    CU(cudaMalloc(&d_starts1, 4096 * 8));
    CU(cudaMalloc(&d_found, 8));
    CU(cudaMalloc(&d_found1, 8));
    CU(cudaMalloc(&d_state, 8));
    CU(cudaMemset(d_found, 0, 8));

    LineMatchEnds m(fwd, d_lines, d_ends, d_ids, cap, d_found);
    m.Begin().Run(lines).End();
    MatchStarts(rev, m, d_starts);
    CU(cudaDeviceSynchronize());
    const uint64_t found = Host(d_found, 1)[0];
    const std::vector<uint32_t> got_lines = Host(d_lines, found), got_ids = Host(d_ids, found);
    const std::vector<uint64_t> got_ends = Host(d_ends, found), got_starts = Host(d_starts, found);

    uint64_t k = 0, mismatches = 0;
    for (uint64_t l = 0; l < n_lines; ++l) {
        const uint64_t b = offs[l], len = offs[l + 1] - 1 - b;
        CU(cudaMemset(d_found1, 0, 8));
        StringMatchEnds one(fwd, d_ends1, d_ids1, 4096, d_found1, d_state);
        one.Begin().Run(d_text + b, len).End();
        const uint64_t f = Host(d_found1, 1)[0];
        if (f > 4096) {
            std::fprintf(stderr, "line %llu: %llu entries\n", (unsigned long long) l, (unsigned long long) f);
            return 2;
        }
        MatchStarts(rev, one, d_text + b, len, 0, d_starts1);
        CU(cudaDeviceSynchronize());
        const std::vector<uint64_t> e1 = Host(d_ends1, f), s1 = Host(d_starts1, f);
        const std::vector<uint32_t> i1 = Host(d_ids1, f);
        for (uint64_t j = 0; j < f; ++j, ++k) {
            const uint64_t want_start = s1[j] == PIRE_GPU_NO_START ? s1[j] : s1[j] + b;
            if (k >= found || got_lines[k] != l || got_ends[k] != e1[j] + b || got_ids[k] != i1[j] || got_starts[k] != want_start)
                ++mismatches;
        }
    }
    if (k != found)
        ++mismatches;
    std::printf("%llu lines, %llu entries: %llu mismatches\n", (unsigned long long) n_lines, (unsigned long long) found,
                (unsigned long long) mismatches);
    for (void* p : {(void*) d_text, (void*) d_offs, (void*) d_lines, (void*) d_ids, (void*) d_ends, (void*) d_starts, (void*) d_ids1,
                    (void*) d_ends1, (void*) d_starts1, (void*) d_found, (void*) d_found1, (void*) d_state})
        cudaFree(p);
    return mismatches ? 1 : 0;
}
