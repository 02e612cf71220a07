// host_check.cpp -- Pire::Gpu::MatchesHost on a device, from plain C++: a CSR batch in host memory, or the lines of
// a text (std::getline offsets with PIRE_GPU_RUN_LINES), against the match bits the caller expects.
//
//   host_check <scanner.pire> <corpus> <offsets.u64> <expected.u8> <flags>
//
// The corpus is read into a buffer of exactly the file's size, so a line batch whose text does not end in '\n' is
// read up to its last byte and no further.  Prints "<n> strings: <k> mismatches".
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iterator>
#include <vector>

#include "pire_gpu.hpp"

namespace {

std::vector<uint8_t> ReadFile(const char* path)
{
    std::ifstream in(path, std::ios::binary);
    if (!in) {
        std::fprintf(stderr, "cannot read %s\n", path);
        std::exit(2);
    }
    return std::vector<uint8_t>(std::istreambuf_iterator<char>(in), std::istreambuf_iterator<char>());
}

} // namespace

int main(int argc, char** argv)
{
    if (argc != 6) {
        std::fprintf(stderr, "usage: %s <scanner.pire> <corpus> <offsets.u64> <expected.u8> <flags>\n", argv[0]);
        return 2;
    }
    const std::vector<uint8_t> image = ReadFile(argv[1]);
    const std::vector<uint8_t> corpus = ReadFile(argv[2]);
    const std::vector<uint8_t> raw = ReadFile(argv[3]);
    const std::vector<uint8_t> expected = ReadFile(argv[4]);
    const unsigned flags = (unsigned) std::strtoul(argv[5], nullptr, 0);
    std::vector<uint64_t> offsets(raw.size() / 8);
    for (size_t i = 0; i < offsets.size(); ++i) {
        uint64_t v = 0;
        for (int b = 7; b >= 0; --b)
            v = (v << 8) | raw[i * 8 + b];
        offsets[i] = v;
    }
    const uint64_t n = offsets.empty() ? 0 : offsets.size() - 1;
    if (expected.size() != n) {
        std::fprintf(stderr, "%zu expected bits for %llu strings\n", expected.size(), (unsigned long long) n);
        return 2;
    }
    try {
        Pire::Gpu::Scanner sc(image.data(), image.size(), 0);
        std::vector<bool> matched;
        Pire::Gpu::MatchesHost(sc, corpus.data(), offsets.data(), n, matched, flags);
        uint64_t bad = 0;
        for (uint64_t i = 0; i < n; ++i)
            bad += matched[i] != (expected[i] != 0);
        std::printf("%llu strings: %llu mismatches\n", (unsigned long long) n, (unsigned long long) bad);
        return bad == 0 ? 0 : 1;
    } catch (const Pire::Gpu::Error& e) {
        std::printf("error %d: %s\n", e.Code, e.what());
        return 1;
    }
}
