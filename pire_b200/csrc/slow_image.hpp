// slow_image.hpp -- host-side ingest of a compiled Pire::SlowScanner.
//
// The byte stream is what SlowScanner::Save() writes and Load/Mmap read (reference pire/scanner_io.cpp:71-156,
// pire/scanners/slow.h:173-201; stream header pire/scanners/common.h:44-78).  A SlowScanner is a non-deterministic
// automaton: its state is a SET of NFA states, stepped whole on each byte.  This file turns the image into bit-set
// tables in the reference's own state numbering, so a set read back is a SlowScanner::State's `flags`.
#pragma once

#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

namespace pire_b200 {

// A compiled SlowScanner in index space.
struct Nfa {
    uint32_t states = 0;       // SlowScanner::Size()
    uint32_t letters = 0;      // SlowScanner::GetLettersCount()
    uint32_t start = 0;        // Locals::start: Initialize() = {start}
    bool empty = false;        // SlowScanner::Empty(): the image is SlowScanner::Null() (slow.h:427-431)
    uint32_t words = 0;        // W = ceil(states / 32): 32-bit words of one set

    std::vector<uint16_t> class_of;  // [kMaxCharUnaligned]: letter of bytes 0..255, Epsilon (257, never stepped) and the marks
    std::vector<uint8_t> finals;     // [states]
    // succ[(l * states + s) * words + w]: the successors of state s on letter l as a bit set (NextTranslated's jump
    // list, slow.h:103-130, duplicates collapsed as its flags.Test does)
    std::vector<uint32_t> succ;
    std::vector<uint32_t> final_mask;   // [words]

    // the set after stepping `cur` (words words; bits at or past `states` ignored) through `symbol` (0..259)
    void Next(const uint32_t* cur, uint32_t symbol, uint32_t* out) const;
    bool Final(const uint32_t* set) const;
};

// Parses the stream.  Returns an empty string on success, else a message.  Rejects what SlowScanner::Load / Mmap reject
// (header, truncation) and, in addition, everything that would become an out-of-bounds table read: a start, jump or
// letter outside the automaton, a jump position list that steps back or points past the image, no states or no
// letters.  The size arithmetic is checked against overflow.
std::string ParseSlowImage(const void* data, size_t size, Nfa* out);

// Stream type of an image header (common.h:33-40: 1 Scanner, 3 SlowScanner, ...), or 0 when `size` is too small for
// a header.
uint32_t ImageType(const void* data, size_t size);

} // namespace pire_b200
