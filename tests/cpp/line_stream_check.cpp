// line_stream_check.cpp -- a text fed from host memory in pieces through include/pire_gpu.hpp's LineStream, from plain
// C++ (no Python).
//
//   line_stream_check <half_final_scanner.pire> <n_lines> <slot_bytes> <piece_bytes> <seed>
//
// A pseudo-random text of lines (some empty, some long, \r\n on some, no final newline) is fed in pieces of
// piece_bytes from pageable memory.  Every frame's offsets, shifted by FirstByte, must continue pire_gpu_split_lines of
// the whole resident text; Runner(sc).Run(frame) and LineMatchEnds on the frame must give the resident text's match
// bits and entries for those lines.  Prints "<n> lines, <m> entries: <k> mismatches".
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

int main(int argc, char** argv)
{
    using namespace Pire::Gpu;
    if (argc != 6) {
        std::fprintf(stderr, "usage: %s <half_final.pire> <n_lines> <slot_bytes> <piece_bytes> <seed>\n", argv[0]);
        return 2;
    }
    const std::vector<char> image = ReadFile(argv[1]);
    const uint64_t want_lines = std::strtoull(argv[2], nullptr, 10);
    const uint64_t slot = std::strtoull(argv[3], nullptr, 10), piece = std::strtoull(argv[4], nullptr, 10);
    uint64_t x = std::strtoull(argv[5], nullptr, 10) * 0x9E3779B97F4A7C15ull + 1;
    auto next = [&x] { x ^= x << 13, x ^= x >> 7, x ^= x << 17; return x >> 32; };
    const char* plants[] = {"error", "fatal", "https://", "GET ", "timeout", "hello  world"};
    std::vector<char> text;
    for (uint64_t l = 0; l < want_lines; ++l) {
        if (l)
            text.push_back('\n');
        const uint64_t len = next() % 7 == 0 ? 0 : next() % 97 == 0 ? 5000 + next() % 20000 : next() % 140;
        const size_t at = text.size();
        for (uint64_t k = 0; k < len; ++k)
            text.push_back((char) (0x20 + next() % 95));
        const char* lit = plants[next() % 6];
        if (len > 20 && next() % 2)
            std::memcpy(&text[at + next() % (len - 13)], lit, std::strlen(lit));
        if (len && next() % 5 == 0)
            text.push_back('\r');
    }

    // the resident answer
    Scanner sc(image.data(), image.size(), 0);
    uint8_t* d_text = nullptr;
    uint64_t *d_offs = nullptr, *d_found = nullptr;
    CU(cudaMalloc(&d_text, text.size() + 1));
    CU(cudaMalloc(&d_offs, (want_lines + 2) * 8));
    CU(cudaMalloc(&d_found, 8));
    if (!text.empty())
        CU(cudaMemcpy(d_text, text.data(), text.size(), cudaMemcpyHostToDevice));
    uint64_t n = 0;
    Check(pire_gpu_split_lines(d_text, text.size(), d_offs, want_lines + 1, &n, 0, nullptr), "pire_gpu_split_lines");
    const std::vector<uint64_t> offs = Host(d_offs, n + 1);
    uint32_t *d_bits = nullptr, *d_lines = nullptr, *d_ids = nullptr;
    uint64_t* d_ends = nullptr;
    const uint64_t cap = 4 * text.size() + 64;
    CU(cudaMalloc(&d_bits, (n / 32 + 1) * 4));
    CU(cudaMalloc(&d_lines, cap * 4));
    CU(cudaMalloc(&d_ids, cap * 4));
    CU(cudaMalloc(&d_ends, cap * 8));
    CU(cudaMemset(d_found, 0, 8));
    Runner(sc).Begin().Run(LineFrame{{d_text, d_offs, 0, n}}).End().Launch(d_bits, nullptr, nullptr);
    LineMatchEnds(sc, d_lines, d_ends, d_ids, cap, d_found).Begin().Run(Batch{d_text, d_offs, 0, n}).End();
    const uint64_t found = Host(d_found, 1)[0];
    const std::vector<uint32_t> bits = Host(d_bits, n / 32 + 1), lines = Host(d_lines, found), ids = Host(d_ids, found);
    const std::vector<uint64_t> ends = Host(d_ends, found);

    // the same text, streamed
    cudaStream_t stream;
    CU(cudaStreamCreate(&stream));
    LineStream ls(0, slot, stream);
    LineStream::Frame f;
    uint32_t *f_bits = nullptr, *f_lines = nullptr, *f_ids = nullptr;
    uint64_t *f_ends = nullptr, *f_found = nullptr;
    CU(cudaMalloc(&f_bits, (n / 32 + 1) * 4));
    CU(cudaMalloc(&f_lines, cap * 4));
    CU(cudaMalloc(&f_ids, cap * 4));
    CU(cudaMalloc(&f_ends, cap * 8));
    CU(cudaMalloc(&f_found, 8));
    uint64_t bad = 0, line = 0, byte = 0, entry = 0;
    for (const char* p = text.data();;) {
        const char* stop = p + std::min<uint64_t>(piece, text.data() + text.size() - p);
        p += ls.Feed(p, stop, stop == text.data() + text.size(), f);
        bad += f.FirstLine != line || f.FirstByte != byte;
        if (f.Count) {
            CU(cudaMemsetAsync(f_found, 0, 8, stream));
            Runner(sc).Begin().Run(f).End().Launch(f_bits, nullptr, nullptr, stream);
            LineMatchEnds(sc, f_lines, f_ends, f_ids, cap, f_found, nullptr, nullptr, stream).Begin().Run(f).End();
            CU(cudaStreamSynchronize(stream));
            const std::vector<uint64_t> fo = Host(f.Offsets, f.Count + 1);
            const std::vector<uint32_t> fb = Host(f_bits, f.Count / 32 + 1);
            const uint64_t k = Host(f_found, 1)[0];
            const std::vector<uint32_t> fl = Host(f_lines, k), fi = Host(f_ids, k);
            const std::vector<uint64_t> fe = Host(f_ends, k);
            for (uint64_t i = 0; i <= f.Count; ++i)
                bad += fo[i] + f.FirstByte != offs[f.FirstLine + i];
            for (uint64_t i = 0; i < f.Count; ++i)
                bad += Bit(fb, i) != Bit(bits, f.FirstLine + i);
            for (uint64_t i = 0; i < k; ++i, ++entry)
                bad += entry >= found || fl[i] + f.FirstLine != lines[entry] || fe[i] + f.FirstByte != ends[entry] ||
                       fi[i] != ids[entry];
        }
        line += f.Count;
        byte += f.Bytes;
        if (p == text.data() + text.size() && (line == n))
            break;
    }
    bad += line != n || entry != found;
    std::printf("%llu lines, %llu entries: %llu mismatches\n", (unsigned long long) n, (unsigned long long) found,
                (unsigned long long) bad);
    return bad != 0;
}
