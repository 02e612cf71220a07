// tests/cpp/slow_check.cpp -- Pire::Gpu::SlowScanner (host concept over the parsed bit-set tables) against the
// reference Pire::SlowScanner built from the same patterns: the reference's own Pire::Step and Pire::Runner templates
// instantiated on both, over texts and seeded random walks with marks, compared state set by state set.  Built and
// run by tests/test_cpp_slow.py where the reference headers exist.  Prints "<n> checked, <k> mismatches".
#include <cstdio>
#include <cstdint>
#include <random>
#include <string>
#include <vector>

#include <pire.h>

#include "pire_gpu.hpp"

namespace {

std::vector<uint32_t> Bits(const Pire::SlowScanner::State& st, size_t words)
{
    std::vector<uint32_t> out(words, 0);
    for (unsigned s : st.states)
        out[s / 32] |= 1u << (s % 32);
    return out;
}

} // namespace

int main()
{
    struct Case {
        const char* pattern;
        size_t distance;
    };
    const Case cases[] = {{"a.{30}$", 0}, {"x.{40}$", 0}, {"(a|b).{20}(c|d).{20}$", 0}, {"foo.{64}bar", 0},
                          {"^.{0,80}error.{200}$", 0}, {"hello\\s+w.+d$", 0}, {"internationalization", 1}};
    const char* texts[] = {"", "a", "....a..............................", "....a...............................",
                           "xx foo" "................................................................" "bar yy",
                           "hello world", "internationalisation", "intrnationalization", "a\nb\n\n"};
    std::mt19937 rng(20261019);
    int bad = 0, checked = 0;
    for (const Case& c : cases) {
        Pire::Fsm fsm = Pire::Lexer(c.pattern).Parse();
        fsm.Surround();
        Pire::SlowScanner ref = fsm.Compile<Pire::SlowScanner>(c.distance);
        Pire::Gpu::SlowScanner mine(ref, /*device*/ -1);
        const size_t words = mine.SetWords();
        if (mine.Size() != ref.Size() || mine.LettersCount() != ref.GetLettersCount() || mine.RegexpsCount() != ref.RegexpsCount()
            || mine.Empty() != ref.Empty() || words != (ref.Size() + 31) / 32) {
            std::printf("%s: sizes differ\n", c.pattern);
            ++bad;
        }
        // Runner(sc).Begin().Run(text).End() through the reference's own templates on both scanners
        for (const char* t : texts) {
            const std::string s(t);
            auto a = Pire::Runner(ref).Begin().Run(s).End();
            auto b = Pire::Runner(mine).Begin().Run(s).End();
            ++checked;
            if (ref.Final(a.State()) != mine.Final(b.State()) || Bits(a.State(), words) != b.State()) {
                std::printf("%s on \"%s\": differs\n", c.pattern, t);
                ++bad;
            }
        }
        // seeded random walks over a small alphabet and both marks, compared after every step
        const char alphabet[] = "abcdefhorx.\n0123456789 ";
        for (int walk = 0; walk < 20; ++walk) {
            Pire::SlowScanner::State a;
            Pire::Gpu::SlowScanner::State b;
            ref.Initialize(a);
            mine.Initialize(b);
            for (int k = 0; k < 300; ++k) {
                const unsigned r = rng() % 64;
                const Pire::Char ch = r == 0 ? Pire::BeginMark : r == 1 ? Pire::EndMark
                                    : r < 4 ? (Pire::Char) (rng() % 256) : (Pire::Char) (unsigned char) alphabet[rng() % (sizeof(alphabet) - 1)];
                Pire::Step(ref, a, ch);
                Pire::Step(mine, b, ch);
                ++checked;
                if (ref.Final(a) != mine.Final(b) || Bits(a, words) != b) {
                    std::printf("%s: walk %d step %d differs\n", c.pattern, walk, k);
                    ++bad;
                    break;
                }
            }
        }
    }
    // SlowScanner::Null(): Empty(), one state, never final
    Pire::SlowScanner null;
    Pire::Gpu::SlowScanner gnull(null, -1);
    Pire::Gpu::SlowScanner::State st;
    gnull.Initialize(st);
    ++checked;
    if (!gnull.Empty() || gnull.Size() != null.Size() || gnull.RegexpsCount() != 0 || gnull.Final(st))
        ++bad;
    std::printf("%d checked, %d mismatches\n", checked, bad);
    return bad ? 1 : 0;
}
