// pair_lines_check.cpp -- two scanners over the lines of a text through include/pire_gpu.hpp, from plain C++ (no
// Python).
//
//   pair_lines_check <first.pire> <second.pire> <n_lines> <seed>
//
// A pseudo-random text of lines (some empty, some of several KiB, \r\n on some, no final newline) is scanned by
// Runner(pair).Begin().Run(frame).End() resident (LineFrame{{d_text, d_offs, 0, n}}) and frame by frame through a
// LineStream with slots smaller than the longest line; each scanner's match bits, masks and states must equal
// Runner(sc).Begin().Run(frame).End() of that scanner alone on the resident text.  A PairRunner with From() starts
// given a LineFrame must throw Error(PIRE_GPU_EINVAL) at Launch.  Prints "<n> lines: <k> mismatches".
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

static bool Bit(const std::vector<uint32_t>& w, uint64_t i) { return (w[i / 32] >> (i % 32)) & 1u; }

struct Outs {
    uint32_t *bits = nullptr, *masks = nullptr, *states = nullptr;
    explicit Outs(uint64_t n)
    {
        CU(cudaMalloc(&bits, (n / 32 + 1) * 4));
        CU(cudaMalloc(&masks, (n + 1) * 4));
        CU(cudaMalloc(&states, (n + 1) * 4));
    }
    Pire::Gpu::RunOutputs Run() const { return Pire::Gpu::RunOutputs{bits, masks, states}; }
};

int main(int argc, char** argv)
{
    using namespace Pire::Gpu;
    if (argc != 5) {
        std::fprintf(stderr, "usage: %s <first.pire> <second.pire> <n_lines> <seed>\n", argv[0]);
        return 2;
    }
    const std::vector<char> image1 = ReadFile(argv[1]), image2 = ReadFile(argv[2]);
    const uint64_t want_lines = std::strtoull(argv[3], nullptr, 10);
    uint64_t x = std::strtoull(argv[4], nullptr, 10) * 0x9E3779B97F4A7C15ull + 1;
    auto next = [&x] { x ^= x << 13, x ^= x >> 7, x ^= x << 17; return x >> 32; };
    const char* plants[] = {"error", "fatal", "https://", "GET ", "timeout", "hello  world", "Hello World"};
    std::vector<char> text;
    for (uint64_t l = 0; l < want_lines; ++l) {
        if (l)
            text.push_back('\n');
        const uint64_t len = next() % 7 == 0 ? 0 : next() % 97 == 0 ? 5000 + next() % 20000 : next() % 140;
        const size_t at = text.size();
        for (uint64_t k = 0; k < len; ++k)
            text.push_back((char) (0x20 + next() % 95));
        const char* lit = plants[next() % 7];
        if (len > 20 && next() % 2)
            std::memcpy(&text[at + next() % (len - 13)], lit, std::strlen(lit));
        if (len && next() % 5 == 0)
            text.push_back('\r');
    }

    Scanner sc1(image1.data(), image1.size(), 0), sc2(image2.data(), image2.size(), 0);
    const ScannerPair pair(sc1, sc2);
    uint8_t* d_text = nullptr;
    uint64_t* d_offs = nullptr;
    CU(cudaMalloc(&d_text, text.size() + 1));
    CU(cudaMalloc(&d_offs, (want_lines + 2) * 8));
    if (!text.empty())
        CU(cudaMemcpy(d_text, text.data(), text.size(), cudaMemcpyHostToDevice));
    uint64_t n = 0;
    Check(pire_gpu_split_lines(d_text, text.size(), d_offs, want_lines + 1, &n, 0, nullptr), "pire_gpu_split_lines");
    const LineFrame whole{{d_text, d_offs, 0, n}};

    // each scanner alone, then the pair, on the resident text
    const Outs a1(n), a2(n), p1(n), p2(n);
    Runner(sc1).Begin().Run(whole).End().Launch(a1.bits, a1.masks, a1.states);
    Runner(sc2).Begin().Run(whole).End().Launch(a2.bits, a2.masks, a2.states);
    Runner(pair).Begin().Run(whole).End().Launch(p1.Run(), p2.Run());
    CU(cudaDeviceSynchronize());
    const Outs* alone[2] = {&a1, &a2};
    const Outs* paired[2] = {&p1, &p2};
    std::vector<uint32_t> bits[2], masks[2], states[2];
    uint64_t bad = 0;
    for (int k = 0; k < 2; ++k) {
        bits[k] = Host(alone[k]->bits, n / 32 + 1);
        masks[k] = Host(alone[k]->masks, n);
        states[k] = Host(alone[k]->states, n);
        bad += Host(paired[k]->bits, (n + 31) / 32) != std::vector<uint32_t>(bits[k].begin(), bits[k].begin() + (n + 31) / 32);
        bad += Host(paired[k]->masks, n) != masks[k];
        bad += Host(paired[k]->states, n) != states[k];
    }

    // the same text streamed through slots smaller than its longest line
    cudaStream_t stream;
    CU(cudaStreamCreate(&stream));
    LineStream ls(0, 4096, stream);
    LineStream::Frame f;
    const Outs f1(n), f2(n);
    uint64_t line = 0;
    for (const char* p = text.data();;) {
        const char* stop = p + std::min<uint64_t>(3000, text.data() + text.size() - p);
        p += ls.Feed(p, stop, stop == text.data() + text.size(), f);
        bad += f.FirstLine != line;
        if (f.Count) {
            Runner(pair).Begin().Run(f).End().Launch(f1.Run(), f2.Run(), stream);
            CU(cudaStreamSynchronize(stream));
            const Outs* got[2] = {&f1, &f2};
            for (int k = 0; k < 2; ++k) {
                const std::vector<uint32_t> fb = Host(got[k]->bits, f.Count / 32 + 1), fm = Host(got[k]->masks, f.Count),
                                            fs = Host(got[k]->states, f.Count);
                for (uint64_t i = 0; i < f.Count; ++i)
                    bad += Bit(fb, i) != Bit(bits[k], f.FirstLine + i) || fm[i] != masks[k][f.FirstLine + i] ||
                           fs[i] != states[k][f.FirstLine + i];
            }
        }
        line += f.Count;
        if (p == text.data() + text.size() && line == n)
            break;
    }
    bad += line != n;

    // lines start from Initialize(): From() starts are refused
    uint32_t* d_starts = nullptr;
    CU(cudaMalloc(&d_starts, (n + 1) * 4));
    try {
        Runner(pair, BatchRunner::From(d_starts), BatchRunner::From(d_starts)).Run(whole).Launch(p1.Run(), p2.Run());
        ++bad;
    } catch (const Error& e) {
        bad += e.Code != PIRE_GPU_EINVAL;
    }
    std::printf("%llu lines: %llu mismatches\n", (unsigned long long) n, (unsigned long long) bad);
    return bad != 0;
}
