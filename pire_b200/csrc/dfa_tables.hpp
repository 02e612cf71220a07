// dfa_tables.hpp -- device table layout for the scan kernels, built on the
// host from a Dfa (pire_image.hpp).
//
// The reference walks  state = row(state)[letter_of[byte]]  with two dependent
// loads per byte (pire/scanners/multi.h:163-192).  On the GPU the walk is bound by
// shared-memory wavefronts, so the layout is chosen to need ONE one-byte shared
// load per input byte on the common path:
//
//  * states are renumbered so that the H <= 255 most frequently visited ("hot")
//    states get ids 0..H-1; id H is the "miss" marker;
//  * hot8[(H+1) rows, kHotStride = 292 bytes apart]: fused byte-indexed rows for hot
//    states, one u8 per (state, byte): the next hot id, or H when the target is a cold
//    state.  Row H maps every byte to H, so a lane that missed keeps running harmlessly
//    to the end of its 16-byte chunk and is then replayed through the full table.
//    The address of an entry is base + 292 * id + byte: one PRMT puts the byte into the
//    low bits of the (256-byte aligned) base -- independent of the state -- and one IMAD
//    (FMA pipe) adds the row, so a step's dependent chain is IMAD -> LDS;
//  * full[states x letters] (u16 when states <= 65536, else u32) + cls[256]:
//    the complete class-indirect table in the new numbering, L2-resident, used
//    only for replays, cold states and the unaligned head/tail bytes;
//  * fin[2][states]: what RunHelper::End()/operator bool/AcceptedRegexps/
//    StateIndex (run.h:376-381, multi.h:143-158,:281-284) report for a string
//    that stops in a given state, precomputed for with_end = 0/1, so the
//    EndMark step and the accept-list walk are one 8-byte load per string;
//  * start[2]: the state after Initialize() and (optionally) Begin()
//    (run.h:369,:375) -- identical for every string, so it is computed once here.
#pragma once

#include <cstdint>
#include <vector>

#include "pire_image.hpp"

namespace pire_b200 {

constexpr uint32_t kMaxHot = 255;
// Bytes from one fused hot row to the next: 256 entries + 36 bytes of padding, so that consecutive rows start
// nine banks apart.  Lanes in different rows then spread over the banks instead of meeting in the 24 banks
// the printable bytes of every row share (host model tools/analyze.cpp, glued ten: 2.44 -> 2.22 wavefronts per
// step plain, 2.23 -> 2.05 with the exit filter).
constexpr uint32_t kHotStride = 292;
// rows are stored in multiples of four so that the table's size stays a multiple of 16 bytes (TMA bulk copy)
inline size_t HotTableBytes(uint32_t hot) { return (size_t) ((hot + 1 + 3) / 4 * 4) * kHotStride; }
constexpr uint32_t kMaxPrivRows = 48;     // lane-private rows incl. the sink (12 quads x 16 KB of shared memory)
constexpr uint32_t kPrivHotRows = 115;    // shared second-tier rows that still fit beside them (116 x 292 B)

struct FinEntry {
    uint32_t result;   // bit31 = Final(), bits 0..30 = StateIndex() in the reference's numbering
    uint32_t mask;     // bit i = regexp id i accepted (ids < 32)
};

struct ScanTables {
    uint32_t states = 0, letters = 0, hot = 0;
    bool wide = false;                       // full table entries are u32
    std::vector<uint32_t> new_of_old, old_of_new;
    std::vector<uint8_t> hot8;               // HotTableBytes(hot): entry of (id, byte) at id * kHotStride + byte
    std::vector<uint8_t> noexit;             // [hot + 1]: 1 = no byte leaves this hot state
    std::vector<uint16_t> cls;               // [256]
    std::vector<uint16_t> full16;
    std::vector<uint32_t> full32;
    std::vector<FinEntry> fin[2];            // [with_end][new id]
    uint32_t start[2] = {0, 0};              // [with_begin] -> new id
    std::vector<uint8_t> flags_new;          // [new id]: bit0 Final, bit1 Dead (prefix scans test them per byte)
    uint32_t end_class = 0;                  // letter class of EndMark (prefix scans step it explicitly)
    uint32_t exit_bitmap0 = ~0u;             // bit (b & 31) set if byte b may leave hot id 0 (kPred filter)
    // LOOK variant (two-byte look-ahead of the exit filter): bit (b & 31) set if byte b leaves hot id 0, or keeps a
    // state entered from hot id 0 from falling back to it.  A lane resting in id 0 reads the table only when this
    // byte AND the next one pass the filter; look_ok = 0 when an exit of id 0 leads to a cold state (the set is
    // then unknown and the variant is not offered).
    uint32_t look_bitmap = ~0u;
    uint64_t look_bitmap64 = ~0ull;          // the same set with 64 slots (slot = b & 63): LOOK64 variant
    bool look_ok = false;
    // Counting (HalfFinalScanner, half_final.h:154-163): hot ids >= first_final_hot are final states
    // (== hot when none is); accept lists in the new numbering as CSR, ids repeated as the image has them.
    uint32_t first_final_hot = 0;
    uint32_t begin_class = 0;                // letter class of BeginMark
    uint32_t initial = 0;                    // new id of Initialize()'s state
    std::vector<uint32_t> acc_begin_new;     // [states + 1]
    std::vector<uint32_t> acc_ids_new;
    // The same lists as packed per-state increments: weights[s * count_words + j] holds, 8 bits each, how
    // often regexps 8j..8j+7 are listed for state s (0 for a non-final state), so TakeAction is one 64-bit
    // add per word.  count_words = 0 when the automaton does not fit (more than 16 regexps, or a regexp
    // listed more than 15 times for one state); the kernel then walks the lists.
    uint32_t count_words = 0;
    std::vector<uint64_t> weights;

    // Lane-private rows (kernel variant PRIV): the first priv_rows-1 hot ids, plus a sink
    // row (id priv_rows-1) that absorbs every transition into a non-private state.  Only
    // bytes 0..127 are covered.  priv_packed[q*128 + b] holds the four entries of quad q
    // (rows 4q..4q+3) for byte b; the kernel replicates each word into all 32 banks so that
    // lane l only ever touches bank l: one wavefront per load, no conflicts by construction.
    uint32_t priv_rows = 0;                  // multiple of 4
    std::vector<uint32_t> priv_packed;       // (priv_rows / 4) * 128
    // The PRIV kernel's second tier: the same fused rows as hot8, cut to the first
    // hot_small ids (what fits in shared memory next to the private region).
    uint32_t hot_small = 0;
    std::vector<uint8_t> hot8_small;         // HotTableBytes(hot_small), same layout
};

// Default hot order: breadth-first from the start states (states near the start
// dominate on text that rarely matches).  Returns old state ids, best first.
std::vector<uint32_t> StaticHotOrder(const Dfa& dfa);

// Hot order from observed visit counts (pire_gpu_scanner_tune): old ids by
// descending count, ties by id; unvisited states are appended in static order.
std::vector<uint32_t> HotOrderFromCounts(const Dfa& dfa, const std::vector<uint64_t>& visits);

// hot_order lists old state ids, most important first; the first
// min(kMaxHot, states, max_hot) become hot.
void BuildScanTables(const Dfa& dfa, const std::vector<uint32_t>& hot_order, uint32_t max_hot, ScanTables* out);

} // namespace pire_b200
