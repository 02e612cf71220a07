// slow_ref.cpp -- a C face over the reference's Pire::SlowScanner, for tests/golden/make_slow_images.py only.
//
// make_slow_images.py compiles this file against the reference tree and the library oracle/build_ref.sh builds
// (oracle/_ref/libpire_ref.so), loads it with ctypes and records the reference's images and answers.  Nothing in the
// product or in the tests links it.
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include <pire.h>
#include <stub/memstreams.h>

namespace {

// The option letters of tests/common.h:40-58: i case-insensitive, u UTF-8, n not surrounded, a & and ~,
// r reversed.
Pire::Fsm Parse(const char* pattern, size_t len, const char* options)
{
    Pire::Lexer lexer;
    Pire::TVector<Pire::wchar32> ucs4;
    bool surround = true, reverse = false;
    for (; options && *options; ++options) {
        if (*options == 'i')
            lexer.AddFeature(Pire::Features::CaseInsensitive());
        else if (*options == 'u')
            lexer.SetEncoding(Pire::Encodings::Utf8());
        else if (*options == 'n')
            surround = false;
        else if (*options == 'a')
            lexer.AddFeature(Pire::Features::AndNotSupport());
        else if (*options == 'r')
            reverse = true;
        else
            throw std::invalid_argument(std::string("Unknown option: ") + *options);
    }
    lexer.Encoding().FromLocal(pattern, pattern + len, std::back_inserter(ucs4));
    lexer.Assign(ucs4.begin(), ucs4.end());
    Pire::Fsm fsm = lexer.Parse();
    if (surround)
        fsm.Surround();
    if (reverse)
        fsm = fsm.Reverse();
    return fsm;
}

uint64_t Emit(const Pire::SlowScanner& sc, void* buf, uint64_t cap)
{
    Pire::BufferOutput out;
    sc.Save(&out);
    const uint64_t n = out.Buffer().Size();
    if (buf && cap >= n)
        std::memcpy(buf, out.Buffer().Data(), n);
    return n;
}

} // namespace

extern "C" {

// Compile<SlowScanner>(distance) of the pattern; *determinable = Fsm::Determine(max_size) succeeded on a copy.
// Returns the image size (the image is written when it fits in cap), 0 on error.
uint64_t slow_ref_compile(const char* pattern, uint64_t len, const char* options, uint64_t distance, uint64_t max_size,
                          int* determinable, void* buf, uint64_t cap)
{
    try {
        Pire::Fsm fsm = Parse(pattern, (size_t) len, options);
        if (determinable) {
            Pire::Fsm copy = fsm;
            *determinable = copy.Determine(max_size) ? 1 : 0;
        }
        return Emit(fsm.Compile<Pire::SlowScanner>(distance), buf, cap);
    } catch (std::exception&) {
        return 0;
    }
}

// The image of SlowScanner::Null() (a default-constructed SlowScanner).
uint64_t slow_ref_null(void* buf, uint64_t cap) { return Emit(Pire::SlowScanner(), buf, cap); }

// Load the image and run Runner(sc[, st_i]) [.Begin()] .Run(string i) [.End()] for every string.  starts: n rows of
// `words` words or null; final_out: n bytes; sets_out: n rows of `words` words (the State's flags).  Returns
// Size(), or 0 when Load throws.
uint64_t slow_ref_run(const void* image, uint64_t size, const uint8_t* corpus, const uint64_t* offsets, uint64_t n,
                      int begin, int end, const uint32_t* starts, uint64_t words, uint8_t* final_out, uint32_t* sets_out,
                      uint64_t* letters_out, int* empty_out)
{
    Pire::SlowScanner sc;
    try {
        Pire::MemoryInput in((const char*) image, (size_t) size);
        sc.Load(&in);
    } catch (std::exception&) {
        return 0;
    }
    const size_t S = sc.Size();
    if (letters_out)
        *letters_out = sc.GetLettersCount();
    if (empty_out)
        *empty_out = sc.Empty() ? 1 : 0;
    for (uint64_t i = 0; i < n; ++i) {
        Pire::SlowScanner::State st;
        sc.Initialize(st);
        if (starts) {
            st.states.clear();
            Pire::BitSet(S).Swap(st.flags);
            for (size_t s = 0; s < S; ++s)
                if (starts[i * words + s / 32] >> (s % 32) & 1) {
                    st.states.push_back((unsigned) s);
                    st.flags.Set(s);
                }
        }
        Pire::RunHelper<Pire::SlowScanner> r = Pire::Runner(sc, st);
        if (begin)
            r.Begin();
        r.Run((const char*) corpus + offsets[i], (const char*) corpus + offsets[i + 1]);
        if (end)
            r.End();
        final_out[i] = sc.Final(r.State()) ? 1 : 0;
        if (sets_out) {
            std::memset(sets_out + i * words, 0, words * 4);
            for (unsigned s : r.State().states)
                sets_out[i * words + s / 32] |= 1u << (s % 32);
        }
    }
    return S;
}

} // extern "C"
