// slow_image.cpp -- see slow_image.hpp.
#include "slow_image.hpp"

#include <cstring>

#include "pire_image.hpp"

namespace pire_b200 {

namespace {

// Stream header, pire/scanners/common.h:44-63.
struct StreamHeader {
    uint32_t magic, version, ptr_size, max_word_size, type, hdr_size;
};
static_assert(sizeof(StreamHeader) == 24, "header layout");

// SlowScanner::Locals on x86-64, slow.h:324-328.
struct SlowLocals {
    uint64_t states, letters, start;
};
static_assert(sizeof(SlowLocals) == 24, "locals layout");

constexpr uint32_t kMagic = 0x45524950u;     // "PIRE", common.h:52
constexpr uint32_t kTypeSlow = 3;            // ScannerIOTypes::SlowScanner, common.h:38
constexpr uint32_t kEpsilon = 257;           // defs.h:62

size_t RoundUp8(size_t v) { return (v + 7) & ~size_t(7); }

// Takes `count` items of `item` bytes at *pos and the padding to 8 behind them (Impl::MapPtr / AlignedLoadArray read
// both, so an image cut inside the padding is refused as Load refuses it); false past the end.
bool Take(size_t size, size_t* pos, uint64_t count, size_t item, const uint8_t** at, const uint8_t* base)
{
    if (count > (size - *pos) / item)
        return false;
    const size_t bytes = RoundUp8((size_t) count * item);
    if (bytes > size - *pos)
        return false;
    *at = base + *pos;
    *pos += bytes;
    return true;
}

} // namespace

uint32_t ImageType(const void* data, size_t size)
{
    if (!data || size < sizeof(StreamHeader))
        return 0;
    StreamHeader h;
    std::memcpy(&h, data, sizeof(h));
    return h.type;
}

std::string ParseSlowImage(const void* data, size_t size, Nfa* out)
{
    *out = Nfa();
    const uint8_t* p = static_cast<const uint8_t*>(data);
    if (!p)
        return "null scanner image";
    if (size < sizeof(StreamHeader) + sizeof(SlowLocals) + 8)
        return "EOF reached while mapping Pire::SlowScanner";                   // common.h:90-92

    StreamHeader h;
    std::memcpy(&h, p, sizeof(h));
    if (h.magic != kMagic || h.ptr_size != 8 || h.max_word_size != 16)
        return "Serialized regexp incompatible with your system";               // common.h:67-68
    if (h.version != 7 && h.version != 6)
        return "You are trying to used an incompatible version of a serialized regexp";   // :69-70
    if (h.type != kTypeSlow || h.hdr_size != sizeof(SlowLocals))
        return "Serialized regexp incompatible with your system";               // :71-76 (not a SlowScanner)
    size_t pos = sizeof(StreamHeader);

    SlowLocals m;
    std::memcpy(&m, p + pos, sizeof(m));
    pos += sizeof(m);
    const bool empty = p[pos] != 0;                                             // scanner_io.cpp:118-120
    pos += 8;

    if (empty) {
        // SlowScanner::Null() = Fsm::MakeFalse().Compile<SlowScanner>(): one state, one letter, no jumps, no finals; the
        // saved Locals are replaced by Null()'s own (Alias, slow.h:381-394), so Size() is 1 whatever the image says
        out->empty = true;
        out->states = 1;
        out->letters = 1;
        out->start = 0;
        out->words = 1;
        out->class_of.assign(kMaxCharUnaligned, 0);
        out->finals.assign(1, 0);
        out->succ.assign(1, 0);
        out->final_mask.assign(1, 0);
        return std::string();
    }

    if (m.states == 0 || m.letters == 0)
        return "slow scanner image has no states or letters";
    if (m.start >= m.states)
        return "slow scanner image: start state outside the automaton";
    // Every table below must lie inside the image, so each count is bounded by `size` before it is multiplied.
    if (m.states > size || m.letters > (size / 8) / m.states)
        return "EOF reached while mapping Pire::SlowScanner";
    const uint64_t cells = m.states * m.letters;

    const uint8_t *letters_p, *finals_p, *pos_p, *jumps_p;
    if (!Take(size, &pos, kMaxChar, 8, &letters_p, p) || !Take(size, &pos, m.states, 1, &finals_p, p)
        || !Take(size, &pos, cells + 1, 8, &pos_p, p))
        return "EOF reached while mapping Pire::SlowScanner";
    uint64_t total;
    std::memcpy(&total, pos_p + cells * 8, 8);
    if (!Take(size, &pos, total, 4, &jumps_p, p))
        return "EOF reached while mapping Pire::SlowScanner";

    out->states = (uint32_t) m.states;
    out->letters = (uint32_t) m.letters;
    out->start = (uint32_t) m.start;
    out->words = (out->states + 31) / 32;
    const uint32_t S = out->states, L = out->letters, W = out->words;

    out->class_of.resize(kMaxCharUnaligned);
    for (uint32_t c = 0; c < kMaxChar; ++c) {
        uint64_t l;
        std::memcpy(&l, letters_p + (size_t) c * 8, 8);
        if (c == kEpsilon)             // filled with 0 and never stepped by a scanner
            l = l < L ? l : 0;
        else if (l >= L)
            return "slow scanner image: letter outside the alphabet";
        if (c < kMaxCharUnaligned)
            out->class_of[c] = (uint16_t) l;
    }

    out->finals.resize(S);
    out->final_mask.assign(W, 0);
    for (uint32_t s = 0; s < S; ++s) {
        out->finals[s] = finals_p[s] != 0;
        if (out->finals[s])
            out->final_mask[s / 32] |= 1u << (s % 32);
    }

    // jumpPos[s * L + l] .. jumpPos[s * L + l + 1] are the jumps of (s, l) (slow.h:108-111); the stream starts at 0
    out->succ.assign((size_t) L * S * W, 0);
    uint64_t prev;
    std::memcpy(&prev, pos_p, 8);
    if (prev != 0)
        return "slow scanner image: jump positions do not start at 0";
    for (uint64_t k = 0; k < cells; ++k) {
        uint64_t next;
        std::memcpy(&next, pos_p + (k + 1) * 8, 8);
        if (next < prev || next > total)
            return "slow scanner image: jump positions step back or past the jumps";
        const uint32_t s = (uint32_t) (k / L), l = (uint32_t) (k % L);
        uint32_t* row = &out->succ[((size_t) l * S + s) * W];
        for (uint64_t j = prev; j < next; ++j) {
            uint32_t t;
            std::memcpy(&t, jumps_p + j * 4, 4);
            if (t >= S)
                return "slow scanner image: jump outside the automaton";
            row[t / 32] |= 1u << (t % 32);
        }
        prev = next;
    }
    return std::string();
}

void Nfa::Next(const uint32_t* cur, uint32_t symbol, uint32_t* out) const
{
    std::vector<uint32_t> next(words, 0);
    const uint32_t l = class_of[symbol];
    for (uint32_t s = 0; s < states; ++s)
        if (cur[s / 32] >> (s % 32) & 1) {
            const uint32_t* row = &succ[((size_t) l * states + s) * words];
            for (uint32_t w = 0; w < words; ++w)
                next[w] |= row[w];
        }
    std::memcpy(out, next.data(), words * 4);
}

bool Nfa::Final(const uint32_t* set) const
{
    for (uint32_t w = 0; w < words; ++w) {
        uint32_t keep = w + 1 < words || states % 32 == 0 ? ~0u : (1u << (states % 32)) - 1;
        if (set[w] & keep & final_mask[w])
            return true;
    }
    return false;
}

} // namespace pire_b200
