// tools/model_look.cpp -- host model of exit filters for the resting state (hot id 0), round 2.
//
// Lanes resting in hot id 0 skip the table read when a filter over the input says the read cannot change
// their state.  Modes:
//   now   : skip iff !F1(b_k)                      F1 = bytes that leave id 0            (round-1 kPred)
//   look  : skip iff !F(b_k) || !F(b_k+1)          F  = F1 + every byte on which a state entered from id 0
//                                                       does not fall back to id 0
//           (a lane that skips an exit byte is "virtually" in id 0: the next byte returns it there anyway)
// For every cheap slot function (what the SHF probe can see) the model reports active lanes and shared-memory
// wavefronts per warp-wide step with the real tables (292-byte rows) over the synthetic corpus.
//
//   model_look <scanner.img> <n_strings> <string_len> [plant ...]
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <functional>
#include <iterator>
#include <string>
#include <vector>

#include "../pire_b200/csrc/dfa_tables.hpp"
#include "../pire_b200/csrc/pire_image.hpp"
#include "../pire_b200/csrc/synth.h"

using namespace pire_b200;

// The LOOKH experiment (round 2, session 44): the filter's 32 slots assigned by slot(b) = mulhi(address + b, mul) & 31,
// `address` = the table's shared-memory address, which the walk adds to every byte anyway.  FoldLookFilter folds an exact
// set (bit b & 31 of exact[b >> 5]) onto those slots; ChooseLookMul searches the multiplier that lets the fewest bytes
// pass (printable ASCII weighted 8:1), over slot widths of 1 to 11 byte values and 32 phases.  The kernel built on it was
// bit-exact and slower (IMAD.HI issues at a quarter of the rate).
static uint32_t FoldLookFilter(const uint32_t exact[8], uint32_t table_address, uint32_t mul)
{
    uint32_t filter = 0;
    for (uint32_t b = 0; b < 256; ++b)
        if (exact[b >> 5] >> (b & 31) & 1u)
            filter |= 1u << ((uint32_t) (((uint64_t) (table_address + b) * mul) >> 32) & 31u);
    return filter;
}

static uint32_t ChooseLookMul(const uint32_t exact[8], uint32_t table_address)
{
    uint32_t best_mul = 0;
    uint32_t best_cost = ~0u;
    const uint64_t phase_step = table_address ? (1ull << 32) / (32ull * table_address) : 0;
    for (uint32_t i = 92; i <= 1024; ++i) {
        const uint64_t alpha = ((uint64_t) i << 32) / 1024;
        for (uint32_t j = 0; j < (phase_step ? 32u : 1u); ++j) {
            const uint64_t m64 = alpha + j * phase_step;
            if (m64 == 0 || m64 > 0xffffffffull)
                continue;
            const uint32_t mul = (uint32_t) m64;
            const uint32_t filter = FoldLookFilter(exact, table_address, mul);
            uint32_t cost = 0;
            for (uint32_t b = 0; b < 256 && cost < best_cost; ++b)
                if (filter >> ((uint32_t) (((uint64_t) (table_address + b) * mul) >> 32) & 31u) & 1u)
                    cost += (b >= 0x20 && b < 0x7f) ? 8 : 1;
            if (cost < best_cost) {
                best_cost = cost;
                best_mul = mul;
            }
        }
    }
    return best_mul;
}

struct Hash {
    std::string name;
    uint32_t slots;
    std::function<uint32_t(uint32_t)> slot;
    std::function<uint32_t(uint32_t)> slot_odd;       // if set: the slot function of the bytes at odd positions
};

static int PassCount(const bool* set, const Hash& h)
{
    std::vector<uint8_t> dirty(h.slots, 0);
    for (uint32_t b = 0; b < 256; ++b)
        if (set[b])
            dirty[h.slot(b)] = 1;
    int pass = 0;
    for (uint32_t b = 0x20; b < 0x7f; ++b)
        pass += dirty[h.slot(b)];
    return pass;
}

int main(int argc, char** argv)
{
    if (argc < 4) {
        std::fprintf(stderr, "usage: model_look image n len [plants...]\n");
        return 2;
    }
    std::ifstream in(argv[1], std::ios::binary);
    std::vector<char> img((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
    Dfa dfa;
    std::string err = ParsePireImage(img.data(), img.size(), &dfa);
    if (!err.empty()) {
        std::fprintf(stderr, "%s\n", err.c_str());
        return 1;
    }
    const uint64_t n = std::strtoull(argv[2], nullptr, 10);
    const uint32_t len = (uint32_t) std::atoi(argv[3]);
    const uint32_t stride = std::getenv("STRIDE") ? std::atoi(std::getenv("STRIDE")) : 292;
    const bool alt = std::getenv("ALT") != nullptr;           // look-ahead on even positions only

    SynthParams sp;
    std::memset(&sp, 0, sizeof(sp));
    sp.seed = 42;
    sp.n_strings = n;
    sp.string_len = len;
    sp.plant_every = 8;
    std::string packed;
    for (int i = 4; i < argc && sp.n_plants < (uint32_t) kMaxPlants; ++i) {
        const char* lit = argv[i];
        sp.plant_off[sp.n_plants] = (uint32_t) packed.size();
        sp.plant_mode[sp.n_plants] = lit[0] == '^' ? 1 : lit[0] == '$' ? 2 : 0;
        packed += lit + (sp.plant_mode[sp.n_plants] ? 1 : 0);
        ++sp.n_plants;
    }
    sp.plant_off[sp.n_plants] = (uint32_t) packed.size();

    std::vector<uint8_t> corpus(n * len);
    const bool mixed = std::getenv("MIXED") != nullptr;       // BASELINE configs[3] text (synth.h SynthMixedCell), fixed length here
    for (uint64_t i = 0; i < n && mixed; ++i)
        for (uint32_t c = 0; c < len / 4; ++c) {
            uint32_t v = SynthMixedCellPlanted(42, 8, i, len, c);
            std::memcpy(&corpus[i * len + 4 * c], &v, 4);
        }
    for (uint64_t i = 0; i < n && !mixed; ++i) {
        uint8_t* dst = &corpus[i * len];
        for (uint32_t w = 0; w < len / 8; ++w) {
            uint64_t v = SynthWord(sp.seed, i, w, len / 8);
            std::memcpy(dst + w * 8, &v, 8);
        }
        uint32_t off;
        int id = SynthPlant(sp, i, &off);
        if (id >= 0)
            std::memcpy(dst + off, packed.data() + sp.plant_off[id], sp.plant_off[id + 1] - sp.plant_off[id]);
    }

    const uint32_t start = dfa.Next(dfa.initial, kBeginMark);
    std::vector<uint64_t> visits(dfa.states, 0);
    for (uint64_t i = 0; i < n; ++i) {
        uint32_t s = start;
        for (uint32_t k = 0; k < len; ++k) {
            ++visits[s];
            s = dfa.Next(s, corpus[i * len + k]);
        }
    }
    std::vector<uint32_t> order = HotOrderFromCounts(dfa, visits);
    ScanTables t;
    BuildScanTables(dfa, order, kMaxHot, &t);
    const uint32_t H = t.hot;
    auto T = [&](uint32_t g, uint32_t b) -> uint32_t { return t.hot8[(size_t) g * kHotStride + b]; };

    bool F1[256], F[256];
    bool look_ok = true;
    for (uint32_t b = 0; b < 256; ++b)
        F1[b] = F[b] = T(0, b) != 0;
    for (uint32_t b = 0; b < 256; ++b)
        if (F1[b]) {
            uint32_t g1 = T(0, b);
            if (g1 == H) {
                look_ok = false;
                continue;
            }
            for (uint32_t c = 0; c < 256; ++c)
                if (T(g1, c) != 0)
                    F[c] = true;
        }
    {
        std::string a, u;
        for (uint32_t b = 0x20; b < 0x7f; ++b) {
            if (F1[b])
                a += (char) b;
            if (F[b])
                u += (char) b;
        }
        std::printf("H %u  F1 (exits of id 0): %zu printable [%s]\n      F: %zu printable [%s] lookahead %s\n", H, a.size(), a.c_str(), u.size(),
                    u.c_str(), look_ok ? "ok" : "DISABLED (an exit of id 0 is cold)");
    }

    std::vector<Hash> hashes;
    hashes.push_back({"exact256", 256, [](uint32_t b) { return b; }});
    hashes.push_back({"b&31", 32, [](uint32_t b) { return b & 31u; }});
    hashes.push_back({"b&63", 64, [](uint32_t b) { return b & 63u; }});
    hashes.push_back({"b&127", 128, [](uint32_t b) { return b & 127u; }});
    // one xorshift round at word level: T(b) = b ^ ((b >> s) & m)  (right) or b ^ ((b << s) & m) (left)
    for (uint32_t slots : {32u, 64u})
        for (int which = 0; which < 2; ++which) {        // 0: best for F1, 1: best for F
            const bool* set = which ? F : F1;
            int best = 1000;
            int bs = 0, bm = 0, bdir = 0;
            for (int dir = 0; dir < 2; ++dir)
                for (int s = 1; s < 8; ++s)
                    for (uint32_t m = 0; m < 256; ++m) {
                        Hash h{"", slots, [=](uint32_t b) { return (b ^ ((dir ? (b << s) : (b >> s)) & m)) & (slots - 1); }};
                        int p = PassCount(set, h);
                        if (p < best) {
                            best = p;
                            bs = s;
                            bm = (int) m;
                            bdir = dir;
                        }
                    }
            char name[64];
            std::snprintf(name, sizeof(name), "xs%u%s(b%s%d&%02x)", slots, which ? "F" : "F1", bdir ? "<<" : ">>", bs, bm);
            const int s = bs, dir = bdir;
            const uint32_t m = (uint32_t) bm;
            hashes.push_back({name, slots, [=](uint32_t b) { return (b ^ ((dir ? (b << s) : (b >> s)) & m)) & (slots - 1); }});
            std::printf("%s passes %d of 95\n", name, best);
        }
    // two rounds (right then left), sampled
    for (uint32_t slots : {32u, 64u}) {
        const bool* set = F;
        int best = 1000;
        uint32_t bp[4] = {0, 0, 0, 0};
        for (int s1 = 1; s1 < 8; ++s1)
            for (uint32_t m1 = 0; m1 < 256; m1 += 1)
                for (int s2 = 1; s2 < 6; ++s2)
                    for (uint32_t m2 = 0; m2 < 64; ++m2) {
                        auto f = [=](uint32_t b) {
                            uint32_t x = b ^ ((b >> s1) & m1);
                            x = (x ^ ((x << s2) & m2)) & 0xff;
                            return x & (slots - 1);
                        };
                        uint64_t dirty = 0;
                        for (uint32_t b = 0; b < 256; ++b)
                            if (set[b])
                                dirty |= 1ull << f(b);
                        int pass = 0;
                        for (uint32_t b = 0x20; b < 0x7f; ++b)
                            pass += (dirty >> f(b)) & 1;
                        if (pass < best) {
                            best = pass;
                            bp[0] = s1; bp[1] = m1; bp[2] = s2; bp[3] = m2;
                        }
                    }
        char name[64];
        std::snprintf(name, sizeof(name), "xs2r%uF(>>%u&%02x,<<%u&%02x)", slots, bp[0], bp[1], bp[2], bp[3]);
        std::printf("%s passes %d of 95\n", name, best);
        const uint32_t s1 = bp[0], m1 = bp[1], s2 = bp[2], m2 = bp[3];
        hashes.push_back({name, slots, [=](uint32_t b) {
                              uint32_t x = b ^ ((b >> s1) & m1);
                              x = (x ^ ((x << s2) & m2)) & 0xff;
                              return x & (slots - 1);
                          }});
    }

    // staircase slots: slot = mulhi(address + b, mul) & 31 -- what ONE multiply-high of (table address + byte) by a
    // constant gives (IMAD.HI, FMA pipe; the LOOKH experiment): runs of neighbouring byte values share a slot, so a filter
    // whose bytes cluster in the code table (digits, neighbouring letters) keeps its false positives next to its members.
    // The multiplier is searched (ChooseLookMul above) for a table at shared address 1024 (MODEL_BASE).
    {
        const uint32_t address = std::getenv("MODEL_BASE") ? (uint32_t) std::atoi(std::getenv("MODEL_BASE")) : 1024u;
        uint32_t exact[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (uint32_t b = 0; b < 256; ++b)
            if (F[b])
                exact[b >> 5] |= 1u << (b & 31);
        const uint32_t mul = ChooseLookMul(exact, address);
        const uint32_t filter = FoldLookFilter(exact, address, mul);
        char name[64];
        std::snprintf(name, sizeof(name), "mulhi32F(mul=%08x)", mul);
        Hash h{name, 32, [=](uint32_t b) { return (uint32_t) (((uint64_t) (address + b) * mul) >> 32) & 31u; }};
        std::printf("%s alpha %.4f passes %d of 95, folded filter %08x (%d slots)\n", name, mul / 4294967296.0, PassCount(F, h), filter,
                    __builtin_popcount(filter));
        hashes.push_back(h);
        Hash half{std::string(name) + " even bytes only", 32, h.slot, [](uint32_t b) { return b & 31u; }};
        hashes.push_back(half);
        // what ONE shift on the ALU pipe gives: slot = (byte + c) >> s, on every position or on the even ones only
        for (uint32_t sh : {1u, 2u})
            for (uint32_t c = 0; c < (1u << sh); ++c) {
                char nm[64];
                std::snprintf(nm, sizeof(nm), "shift32((b+%u)>>%u)", c, sh);
                auto fn = [=](uint32_t b) { return ((b + c) >> sh) & 31u; };
                hashes.push_back({nm, 32, fn});
                hashes.push_back({std::string(nm) + " even bytes only", 32, fn, [](uint32_t b) { return b & 31u; }});
            }
    }

    for (const Hash& h : hashes) {
        std::vector<uint8_t> f1(h.slots, 0), ff(h.slots, 0), ffo(h.slots, 0);
        for (uint32_t b = 0; b < 256; ++b) {
            if (F1[b])
                f1[h.slot(b)] = 1;
            if (F[b])
                ff[h.slot(b)] = 1;
            if (F[b] && h.slot_odd)
                ffo[h.slot_odd(b)] = 1;
        }
        // filter of a byte at position k (look mode): positions alternate between the two slot functions when slot_odd is set
        auto passes = [&](uint32_t b, uint32_t k) -> bool { return (h.slot_odd && (k & 1)) ? ffo[h.slot_odd(b)] != 0 : ff[h.slot(b)] != 0; };
        uint64_t steps = 0, wf[2] = {0, 0}, act[2] = {0, 0}, nonzero[2] = {0, 0};
        uint64_t mismatch = 0;
        for (uint64_t base = 0; base + 32 <= n; base += 32) {
            // mode 0 = now, mode 1 = look; g = register state (hot id or H), full = true state
            uint32_t g[2][32], full[32];
            for (int l = 0; l < 32; ++l) {
                full[l] = t.start[1];
                g[0][l] = g[1][l] = full[l] < H ? full[l] : H;
            }
            for (uint32_t k = 0; k < len; ++k) {
                uint32_t words[2][32][4];
                int cnt[2][32];
                std::memset(cnt, 0, sizeof(cnt));
                for (int l = 0; l < 32; ++l) {
                    const uint8_t b = corpus[(base + l) * len + k];
                    const bool last = k + 1 == len;
                    const uint8_t nb = last ? 0 : corpus[(base + l) * len + k + 1];
                    for (int mode = 0; mode < 2; ++mode) {
                        uint32_t& gg = g[mode][l];
                        bool need;
                        if (mode == 0)
                            need = gg != 0 || f1[h.slot(b)];
                        else if (alt && (k & 1))
                            need = gg != 0 || ff[h.slot(b)];            // ALT: odd positions use the byte's own filter only
                        else
                            need = gg != 0 || (passes(b, k) && (last || !look_ok || passes(nb, k + 1)));
                        nonzero[mode] += gg != 0;
                        if (need) {
                            const uint32_t addr = gg * stride + b;
                            const uint32_t word = addr >> 2, bank = word & 31;
                            bool seen = false;
                            for (int q = 0; q < cnt[mode][bank] && q < 4; ++q)
                                seen = seen || words[mode][bank][q] == word;
                            if (!seen) {
                                if (cnt[mode][bank] < 4)
                                    words[mode][bank][cnt[mode][bank]] = word;
                                ++cnt[mode][bank];
                            }
                            ++act[mode];
                            // cold lanes: keep it simple, follow the true state (the kernel replays them)
                            gg = gg == H ? H : T(gg, b);
                        }
                    }
                    full[l] = t.wide ? t.full32[(size_t) full[l] * t.letters + t.cls[b]] : t.full16[(size_t) full[l] * t.letters + t.cls[b]];
                    for (int mode = 0; mode < 2; ++mode)
                        if (g[mode][l] == H || full[l] >= H)
                            g[mode][l] = full[l] < H ? full[l] : H;       // replay resolves cold excursions
                }
                for (int mode = 0; mode < 2; ++mode) {
                    int w = 0;
                    for (int bnk = 0; bnk < 32; ++bnk)
                        w = std::max(w, cnt[mode][bnk]);
                    wf[mode] += w;
                }
                ++steps;
            }
            for (int l = 0; l < 32; ++l)
                for (int mode = 0; mode < 2; ++mode)
                    mismatch += (g[mode][l] == H ? full[l] : g[mode][l]) != full[l];
        }
        std::printf("%-28s now: %.3f wf %.2f act %.2f nz | look: %.3f wf %.2f act %.2f nz | end-state mismatches %llu\n", h.name.c_str(),
                    (double) wf[0] / steps, (double) act[0] / steps, (double) nonzero[0] / steps, (double) wf[1] / steps, (double) act[1] / steps,
                    (double) nonzero[1] / steps, (unsigned long long) mismatch);
    }
    return 0;
}
