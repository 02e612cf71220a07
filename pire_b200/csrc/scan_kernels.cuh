// scan_kernels.cuh -- launch interface between the C ABI (capi.cu) and the
// sm_90a kernels (scan_kernels.cu).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "dfa_tables.hpp"
#include "synth.h"

namespace pire_b200 {

struct DeviceFin {
    uint32_t result;    // bit31 Final, low bits StateIndex (reference numbering)
    uint32_t mask;      // accepted regexp ids < 32
};

// Everything a scan launch reads.  Device pointers.
struct ScanArgs {
    const uint8_t* corpus;
    const uint64_t* offsets;     // CSR (n+1) or nullptr
    uint32_t trim;               // CSR only: bytes dropped from the end of every string (1 = the newline of a line)
    const uint32_t* order;       // generic kernel: lane i scans string order[i] (length-binned launch), or nullptr
    unsigned int* work_counter;  // with `order`: units are claimed longest-first from this counter
    const uint32_t* split_count; // with `order`, or null: the first *split_count entries of `order` belong to the split kernel
    unsigned int* split_counter; // split kernel: strings are claimed from this counter
    uint32_t split_prefetch;     // split kernel: 32-byte blocks between a lane's walk and its L2 prefetch (0 = none)
    uint64_t fixed_len;          // used when offsets == nullptr
    uint64_t n;                  // strings
    const uint8_t* hot8;         // HotTableBytes(hot) bytes (rows kHotStride apart), 16-byte aligned
    const uint8_t* noexit;       // hot+1 bytes
    const uint16_t* cls;         // 256
    const void* full;            // states*letters, u16 or u32
    const DeviceFin* fin;        // [states] for the chosen with_end
    uint32_t hot;                // H
    uint32_t letters;
    uint32_t wide;               // full is u32
    uint32_t start;              // state after Initialize()[+Begin()], new numbering
    uint32_t exit_bitmap0;       // 32-slot exit bitmap of hot id 0, slot = byte & 31
    uint32_t look_bitmap;        // LOOK variant: 32-slot look-ahead filter (dfa_tables.hpp), slot = byte & 31
    uint64_t look_bitmap64;      // LOOK64 variant: the same filter with 64 slots, slot = byte & 63
    uint32_t uniform;            // prefix / count kernels: fixed length, a multiple of 32 bytes, corpus 32-byte aligned
    uint32_t opaque_zero;        // always 0; the LOOK kernels multiply by it to pin an instruction behind the walk
    const uint32_t* priv_packed; // (priv_rows/4)*128 words, PRIV variant
    uint32_t priv_rows;
    const uint8_t* hot8_small;   // PRIV variant's second tier: HotTableBytes(hot_small)
    uint32_t hot_small;
    uint32_t* match_bits;        // may be null
    uint32_t* accept_masks;      // may be null
    uint32_t* state_idx;         // may be null
    unsigned long long* visits;  // tune kernel only: per-state visit counters (new numbering)
    const uint8_t* flags;        // prefix kernels: [states] bit0 Final, bit1 Dead (new numbering)
    uint32_t end_class;          // prefix kernels: letter class of EndMark
    uint32_t through_end;        // prefix kernels: step EndMark after the bytes
    uint32_t* prefix_len;        // prefix kernels: n words, 0xFFFFFFFF = no accepted prefix
    // counting kernel (HalfFinalScanner::TakeAction, half_final.h:154-163)
    const uint32_t* acc_begin;   // [states + 1] CSR of accept lists, new numbering
    const uint32_t* acc_ids;
    uint32_t first_final_hot;    // hot ids >= this are final states
    uint32_t begin_class;        // letter class of BeginMark
    uint32_t initial;            // Initialize()'s state, new numbering
    uint32_t with_begin;         // step BeginMark first (with_end == through_end)
    uint32_t regexps;            // counters per string (>= 1)
    uint32_t* counts;            // n * regexps words, zeroed by the caller
    uint32_t lines_turn;         // lines kernel: chunks per lane between two hand-outs of lines
    uint32_t lines_min_idle;     // lines kernel: waiting lanes needed for a hand-out
    const uint64_t* weights;     // [states * count_words] packed per-state increments, or null
    uint32_t count_words;        // 0 = walk the accept lists, 1..2 = packed increments
    uint32_t count_always;       // final states are frequent: count every chunk, skip the look-ahead pass
    // one string over the grid (pire_gpu_run_string): corpus, fixed_len = its bytes
    const uint32_t* start_idx;   // the start as a StateIndex (reference numbering) in device memory, or null: `start`
    const uint32_t* new_of_old;  // [states]: reference numbering -> new
    uint32_t states;             // Size(): a start_idx at or above it is out of range
    uint32_t* string_ends;       // scratch: 2 x warps of the grid, each warp's end state per stitching round
    unsigned int* string_rounds; // scratch: 3 counters of changed warps, zeroed before the launch
    // per-string starts (pire_gpu_run_batch_from): string i starts from the StateIndex starts[i] (reference numbering),
    // mapped through new_of_old, BeginMark stepped when with_begin; one at or above `states` reports (0, 0, 0xFFFFFFFF).
    // starts may be state_idx: every kernel reads string i's start before it writes string i's state
    const uint32_t* starts;      // n words, or null: every string starts from `start`
    // counting one string over the grid (pire_gpu_count_string): the counts are added to counts64 (max(1, regexps) words);
    // counting a batch from given states (pire_gpu_count_batch_from): n rows of max(1, regexps) words, row i string i's
    unsigned long long* counts64;
    uint32_t count_rows;         // 1: every warp sums into a row of u32 in shared memory first; 0: straight into counts64
    // where the matches end in one string over the grid (pire_gpu_match_ends_string): the call's entry k goes to index
    // *found + k of ends / ids when that is below ends_capacity; *found is read once and advanced by the call's total
    uint64_t* ends;              // ends_base + bytes consumed when a final state was entered, or null
    uint32_t* ids;               // the regexp id of each entry, or null
    uint64_t ends_capacity;      // entries of ends / ids
    unsigned long long* found;   // one word, read and added to
    uint64_t ends_base;          // position of the text's first byte in the caller's numbering
    unsigned long long* string_sums; // scratch: each CTA's number of entries
    // where the matches end in a batch of streams (pire_gpu_match_ends_batch_from): ends, ids, ends_capacity and found as
    // above (ends_base 0), string i's entries in the slice [entry_first[i], entry_first[i + 1]), its positions from pos[i] on
    uint32_t* strings;           // the string index of each entry, or null
    uint64_t* pos;               // n words: each string's first position, advanced by its length; or null (all 0)
    unsigned long long* entry_counts;      // scratch, n + 1: *found as the call found it, then each string's entries
    const unsigned long long* entry_first; // scratch, n + 1: the inclusive sum of entry_counts
    uint32_t* last_states;       // scratch, n: each string's state before EndMark, new numbering (0xFFFFFFFF: unknown start)
    // where the matches start (pire_gpu_match_starts_*): entries [*entries_first, min(*entries_found, ends_capacity)) of
    // entry_strings / entry_ends / entry_ids; string i's window is [w - len_i, w) with w = window_end[i], or ends_base +
    // len_i when that is null.  An entry's walk goes left from its end to the window start (or max_back bytes), with
    // EndMark first (with_end, entries at the window's end only) and BeginMark last (with_begin, at the window start only).
    const unsigned long long* entries_first;   // or null: 0
    const unsigned long long* entries_found;
    const uint32_t* entry_strings;   // or null: every entry belongs to string 0
    const uint64_t* entry_ends;
    const uint32_t* entry_ids;       // or null: Final() instead of one regexp
    const uint64_t* window_end;
    uint32_t with_end;               // EndMark for entries at their window's end
    uint64_t max_back;               // 0 = no bound
    const uint32_t* live;            // ScanTables::live, live_words per state
    uint32_t live_words;
    uint64_t* match_starts;          // per entry: the leftmost start, or ~0
    uint8_t* match_open;             // per entry, or null: the walk reached its lower bound still live
    unsigned long long* group_counter;   // scratch word, zeroed: groups of 32 entries handed out so far
};

struct LaunchPlan {
    int block = 0;
    int grid = 0;
    size_t shared = 0;
};

enum ScanVariant {
    kVariantPlain = 1,
    kVariantPred = 2,
    kVariantPriv = 3,
    kVariantLook = 4,
    kVariantLook64 = 5,
    kVariantLook1 = 6,
    kVariantLookRing1 = 7
};
constexpr int kVariantSlots = 8;      // size of per-variant arrays (variant ids are 1-based)

size_t ScanSharedBytes(uint32_t hot, uint32_t priv_rows);
cudaError_t PrepareScanKernels(int device);                       // raises the dynamic smem limit
// starts: the plan of the kernel a launch with a.starts runs (the same shape as without; PRIV has no such kernel)
cudaError_t PlanScan(int device, uint32_t hot, uint32_t hot_small, uint32_t priv_rows, int variant, bool uniform, LaunchPlan* plan,
                     bool starts = false);
// a.starts selects the kernels that start every string from its own state
cudaError_t LaunchScan(const ScanArgs& a, int variant, bool uniform, const LaunchPlan& plan, cudaStream_t stream);
// CSR batches of short strings (lines of text): lanes pull strings dynamically; a.match_bits must be zeroed
cudaError_t LaunchLines(const ScanArgs& a, int variant, int device, cudaStream_t stream);
// length-ordered CSR batches: the leading long strings, one per warp; sets *a.split_count, which the generic launch honours
cudaError_t LaunchSplit(const ScanArgs& a, int variant, int device, cudaStream_t stream);
// one string (a.corpus, a.fixed_len bytes) over the whole grid, cooperatively launched; a.with_begin / a.begin_class
// step BeginMark from *a.start_idx when that is given
cudaError_t LaunchString(const ScanArgs& a, int variant, int device, cudaStream_t stream);
// HalfFinalScanner counts of one string over the whole grid (CountStringKernel): LaunchString's grid and pieces, the
// counting fields of LaunchCount, a.counts64 added to; a.start_idx / a.with_begin as in LaunchString
cudaError_t LaunchCountString(const ScanArgs& a, int device, cudaStream_t stream);
// the largest max(1, regexps) for which LaunchCountString keeps a row of counters per warp in shared memory
constexpr uint32_t kCountRowsMax = 256;
// Every TakeAction of HalfFinalScanner on one string over the whole grid (MatchEndsStringKernel): LaunchString's grid and
// pieces, SetCounting's accept lists, the entries in walk order from index *a.found on, *a.found advanced by their number
cudaError_t LaunchMatchEndsString(const ScanArgs& a, int device, cudaStream_t stream);
cudaError_t LaunchVisitCount(const ScanArgs& a, cudaStream_t stream);
// prefix (left to right) or suffix (right to left) scan; a.with_begin/begin_class name the mark stepped first,
// a.through_end/end_class the mark stepped last
cudaError_t LaunchPrefix(const ScanArgs& a, bool shortest, bool reverse, int device, cudaStream_t stream);
// HalfFinalScanner counts of a batch, one string per lane: into a.counts (n rows of u32, zeroed by the caller), or with
// `from` (pire_gpu_count_batch_from) added to a.counts64 (n rows of u64), every string from a.starts[i] when a.starts is
// given, its last state reported in a.match_bits / a.state_idx through a.fin
cudaError_t LaunchCount(const ScanArgs& a, int device, cudaStream_t stream, bool from = false);
// Every TakeAction of HalfFinalScanner on each string of a batch (MatchEndsBatchKernel): LaunchCount's walk with
// `from`, string i's entries from index *a.found + (the entries of strings 0..i-1) on, placed by a scan over the strings;
// then match bits, states and a.pos as LaunchCount's, and *a.found advanced by the call's total
cudaError_t LaunchMatchEndsBatch(const ScanArgs& a, int device, cudaStream_t stream);
// The leftmost start of every match-ends entry (MatchStartsKernel): one entry per lane, walked leftwards through a
// reversed scanner from its end, groups of 32 entries handed to warps of a persistent grid
cudaError_t LaunchMatchStarts(const ScanArgs& a, int device, cudaStream_t stream);
// d_order <- string indices, longest half-octave length bucket first, corpus order inside a bucket (stable CUB radix sort).
// stream-ordered scratch from the library's own per-device pool (see scan_kernels.cu)
cudaError_t ScratchAlloc(void** out, size_t bytes, cudaStream_t stream);
cudaError_t LengthOrder(const uint64_t* d_offsets, uint64_t n, uint32_t* d_order, cudaStream_t stream);
// Line starts of a newline-delimited text (std::getline semantics): d_offsets[0..n_lines], line i =
// text[off[i] .. off[i+1] - 1).  *n_lines is written on the host after a stream synchronise.
cudaError_t SplitLines(const uint8_t* d_text, uint64_t n_bytes, uint64_t* d_offsets, uint64_t capacity, uint64_t* n_lines,
                       cudaStream_t stream);
cudaError_t LaunchSynth(const SynthParams& p, const char* d_plants, uint8_t* d_out, cudaStream_t stream);

cudaError_t LaunchSynthMixedLengths(uint64_t seed, uint64_t first, uint64_t n, uint64_t* d_lengths, cudaStream_t stream);
cudaError_t LaunchSynthMixedFill(uint64_t seed, uint32_t plant_every, uint64_t first, uint64_t n, const uint64_t* d_offsets,
                                 uint8_t* d_out, cudaStream_t stream);

// out[i * words + w] = table[state_idx[i] * words + w] (a state index outside the table yields zeros)
cudaError_t LaunchAcceptGather(const uint32_t* d_table, uint32_t states, uint32_t words, const uint32_t* d_state_idx, uint64_t n,
                               uint32_t* d_out, cudaStream_t stream);

uint64_t KernelLaunchCount();

} // namespace pire_b200
