/* pire_b200.h -- C ABI of the GPU-native (H100, sm_90a) Pire scan path.
 *
 * The reference (yandex/pire) has no plugin/FFI layer: its seam is the
 * compile-time "Scanner concept" consumed by the templates of pire/run.h
 * (SURVEY.md 8(b)).  This header is the boundary a maintainer binds instead:
 * every entry point names the reference interface it replaces.  Signatures use
 * plain pointers and sizes only; device buffers are caller-owned CUDA pointers.
 *
 * Compiled automata cross the boundary as the byte stream written by the
 * reference's own  Pire::Scanner::Save()  (pire/scanners/multi.h:557-573), so
 * the regex front end (Lexer -> Fsm -> Compile / Scanner::Glue) stays on the
 * host, unchanged.  See INTEGRATION.md for the reference-side binding and
 * include/pire_gpu.hpp for the C++ mirror of Scanner / Runner / Matches.
 *
 * All functions return 0 on success or a negative pire_gpu_status; the text of
 * the last error on the calling thread is available from pire_gpu_last_error().
 * The run path of the reference never throws and returns no status
 * (pire/run.h); here bad arguments and CUDA failures are reported instead of
 * being undefined behaviour.
 */
#ifndef PIRE_B200_H
#define PIRE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pire_gpu_scanner pire_gpu_scanner;

typedef enum pire_gpu_status {
    PIRE_GPU_OK = 0,
    PIRE_GPU_EINVAL = -1,      /* bad argument */
    PIRE_GPU_EIMAGE = -2,      /* scanner image rejected (what Scanner::Load/Mmap throw, multi.h:252-272) */
    PIRE_GPU_ECUDA = -3,       /* CUDA runtime error (message holds cudaGetErrorString) */
    PIRE_GPU_ENODEVICE = -4,   /* no usable CUDA device: the scan path has NO CPU fallback */
    PIRE_GPU_EUNSUPPORTED = -5
} pire_gpu_status;

/* Run flags: which of RunHelper's mark steps surround the bytes (run.h:375-376).
 * Runner(sc).Begin().Run(p,n).End() == BEGIN|END; the free function
 * Pire::Matches(sc,b,e) (run.h:396-400) steps neither mark == 0. */
enum {
    PIRE_GPU_RUN_BEGIN = 1u,
    PIRE_GPU_RUN_END = 2u,
    /* CSR offsets come from pire_gpu_split_lines: string i ends one byte before offsets[i+1]
     * (its newline).  Accepted by every entry point that takes CSR offsets. */
    PIRE_GPU_RUN_LINES = 4u
};

/* Kernel variants (pire_gpu_scanner_set_variant). */
enum {
    PIRE_GPU_VARIANT_AUTO = 0,
    PIRE_GPU_VARIANT_PLAIN = 1,    /* one shared-memory load per byte, unconditional */
    PIRE_GPU_VARIANT_PRED = 2,     /* load predicated off while the resident state self-loops */
    PIRE_GPU_VARIANT_PRIV = 3,     /* hottest rows replicated per bank: conflict-free loads (fixed-length ASCII-heavy batches) */
    PIRE_GPU_VARIANT_LOOK = 4,     /* PRED with one byte of look-ahead: a resting lane reads the table only when this byte and
                                      the next can both matter (the device analogue of the ExitMasks skip loop,
                                      multi.h:966-989); fixed-length batches, PRED otherwise */
    PIRE_GPU_VARIANT_LOOK64 = 5,   /* LOOK with a 64-slot filter (one more FMA-pipe instruction per byte, fewer false passes) */
    PIRE_GPU_VARIANT_LOOK1 = 6,    /* LOOK walks two strings per lane on fixed-length batches (the second string's step fills
                                      the latency of the first one's table read); LOOK1 is the same filter with one string per
                                      lane -- the shape for batches too small to give every resident warp two units */
    PIRE_GPU_VARIANT_LOOK_RING1 = 7, /* LOOK1's walk, one string per lane, fed from a ring in shared memory that keeps two
                                      more 32-byte blocks of every string in flight (fixed-length batches; the CSR
                                      look-ahead kernel otherwise) */
    PIRE_GPU_VARIANT_SLOTS = 8    /* length of per-variant arrays indexed by variant id */
};

typedef struct pire_gpu_info {
    uint32_t states;           /* Scanner::Size()          multi.h:134 */
    uint32_t letters;          /* Scanner::LettersCount()  multi.h:140 */
    uint32_t regexps;          /* Scanner::RegexpsCount()  multi.h:139 */
    uint32_t initial;          /* StateIndex(Initialize()) multi.h:161,:281 */
    uint32_t empty;            /* Scanner::Empty()         multi.h:135 */
    uint32_t hot_rows;         /* rows of the shared-memory table */
    uint32_t variant;          /* kernel variant in use */
    uint32_t tuned;            /* 1 after pire_gpu_scanner_tune */
    uint64_t table_bytes;      /* device bytes of the complete (L2-resident) table */
    uint64_t shared_bytes;     /* dynamic shared memory per CTA */
    int32_t  device;           /* CUDA device, or -1 for a host-only handle */
    uint32_t reserved;
} pire_gpu_info;

/* ---- scanner lifetime -----------------------------------------------------
 * Replaces: Scanner::Load / Scanner::Mmap (multi.h:244-279,:575-599) followed
 * by taking the address of the scanner for Runner() (run.h:388-389).
 * `image` is the Scanner::Save() stream of a Pire::Scanner (Relocatable; both
 * ExitMasks<2> and NoShortcuts variants are accepted).  The handle owns device
 * copies of its tables and does not retain `image`.  device >= 0 selects the
 * CUDA device; device == -1 builds a host-only handle (tables + the host
 * accessors below; every run entry point then fails with PIRE_GPU_ENODEVICE).
 * A handle is immutable after create/tune: run_batch is re-entrant across
 * streams, like a const Scanner shared between threads (SURVEY.md 8(b)). */
int  pire_gpu_scanner_create(const void* image, size_t size, int device, pire_gpu_scanner** out);
void pire_gpu_scanner_destroy(pire_gpu_scanner* sc);
int  pire_gpu_scanner_info(const pire_gpu_scanner* sc, pire_gpu_info* out);
int  pire_gpu_scanner_set_variant(pire_gpu_scanner* sc, uint32_t variant);
int  pire_gpu_scanner_set_max_hot(pire_gpu_scanner* sc, uint32_t max_hot_rows);

/* ---- the hot path -----------------------------------------------------------
 * Replaces, for a whole batch of strings at once:
 *     Pire::Runner(sc).Begin().Run(ptr, len).End()          run.h:365-392
 *     -> operator bool / Final()                            run.h:380-381, multi.h:143
 *     -> AcceptedRegexps(state)                             multi.h:149-158
 *     -> StateIndex(state)                                  multi.h:281-284
 * String i is d_corpus[d_offsets[i] .. d_offsets[i+1])  (CSR, n+1 offsets), or,
 * when d_offsets == NULL, d_corpus[i*fixed_len .. (i+1)*fixed_len).  Empty
 * strings are legal (pire_ut.cpp NullPointer); n == 0 is a no-op.
 * Outputs (each may be NULL):
 *   d_match_bits    ceil(n/32) words; bit (i%32) of word i/32 = Final();
 *                   bits past n in the last word are 0
 *   d_accept_masks  n words; bit r = regexp id r in AcceptedRegexps (r < 32)
 *   d_state_idx     n words; StateIndex() of the last state, reference numbering
 * All pointers are device pointers on the handle's device; the launch is
 * asynchronous on `stream` (a cudaStream_t passed as void*; NULL = default).
 * Side effect shared by every entry point that takes a handle, a communicator or a
 * `device` argument: the device becomes the calling thread's current CUDA device
 * (cudaSetDevice) and stays so on return; a caller that works with several devices
 * from one thread re-selects its own afterwards. */
int pire_gpu_run_batch(const pire_gpu_scanner* sc,
                       const uint8_t* d_corpus, const uint64_t* d_offsets,
                       uint64_t fixed_len, uint64_t n, uint32_t flags,
                       uint32_t* d_match_bits, uint32_t* d_accept_masks, uint32_t* d_state_idx,
                       void* stream);

/* Length-binned form of pire_gpu_run_batch for batches of very unequal strings
 * (BASELINE config 4: 16 B .. 64 KiB).  One string per lane means a warp runs as
 * long as its longest string; with `d_order` (a permutation of 0..n-1 from
 * pire_gpu_length_order: longest half-octave length bucket first, corpus order
 * inside a bucket so that a warp's lanes read neighbouring addresses) warps get
 * strings of similar length and claim them longest-first.  Results are still
 * indexed by the original string number.
 * CSR batches only; n < 2^32. */
int pire_gpu_length_order(const uint64_t* d_offsets, uint64_t n, uint32_t* d_order, int device, void* stream);
int pire_gpu_run_batch_ordered(const pire_gpu_scanner* sc,
                               const uint8_t* d_corpus, const uint64_t* d_offsets, const uint32_t* d_order,
                               uint64_t n, uint32_t flags,
                               uint32_t* d_match_bits, uint32_t* d_accept_masks, uint32_t* d_state_idx,
                               void* stream);

/* One long string with the whole GPU.  Replaces, for one string resident in HBM,
 *     Pire::Runner(sc[, st]) [.Begin()] .Run(d_text, d_text + n_bytes) [.End()]        run.h:365-392
 * (the shape of tools/bench/bench.cpp:241-254 and samples/blacklist: a whole file as one string).  The string is cut
 * into one piece per lane of the persistent grid; the pieces are walked at once and stitched exactly (DESIGN.md 4).
 *   Input   d_text[0 .. n_bytes), any length (0 included; d_text may then be NULL), any alignment, past 4 GiB too.
 *   flags   PIRE_GPU_RUN_BEGIN and/or PIRE_GPU_RUN_END; anything else is PIRE_GPU_EINVAL, as is a NULL d_text with
 *           n_bytes > 0.
 *   Start   d_start == NULL: Initialize().  Otherwise d_start points to ONE device word holding a StateIndex in the
 *           reference's numbering (Runner(sc, st), run.h:391-392); BEGIN steps BeginMark from that state.  A start
 *           >= Size() reads no table and yields match 0, mask 0 and state 0xFFFFFFFF (pire_gpu_accept_sets treats that
 *           state as empty, too).
 *   Chain   the d_state_idx of a call made without END is the d_start of the next call -- how a text that arrives in
 *           chunks is scanned: BEGIN on the first call, END on the last, every call in between with neither.
 *           d_state_idx may be the same word as d_start.
 *   Output  as pire_gpu_run_batch with n = 1, each may be NULL: d_match_bits[0] (the whole word: bit 0 = Final(), the
 *           others 0), d_accept_masks[0], d_state_idx[0] (StateIndex of the last state, after End() with END).  Nothing
 *           else is written.
 * Asynchronous on `stream`; re-entrant across streams on one handle (its scratch is per call and stream-ordered).
 * Results are bit-exact with pire_gpu_run_batch on the same bytes (CSR, n = 1).  A host-only handle gets
 * PIRE_GPU_ENODEVICE.  Worst case: when the walks of the pieces from the guessed state never fall together with the
 * true walk, the string is walked about as fast as one lane walks it alone.  That is the case for the parity of a run
 * of a's, and for a scanner that remembers a match until the end of the string (a surrounded glued scanner) when the
 * text has one early match and no more, or when the guess was tuned on text with matches and the text has none
 * (DESIGN.md 4). */
int pire_gpu_run_string(const pire_gpu_scanner* sc, const uint8_t* d_text, uint64_t n_bytes, uint32_t flags,
                        const uint32_t* d_start,
                        uint32_t* d_match_bits, uint32_t* d_accept_masks, uint32_t* d_state_idx, void* stream);

/* A batch of streams resumed where each one stopped.  Replaces, for every string i of a batch,
 *     Pire::Runner(sc, st_i) [.Begin()] .Run(string i) [.End()]                            run.h:365-392
 * (many texts arriving in pieces at once -- connections, log tails, files read block by block -- each carried on from
 * the state its last piece ended in).
 *   Batch   as pire_gpu_run_batch: CSR (d_offsets) or fixed length.  d_order may be NULL; when given it has the
 *           meaning of pire_gpu_run_batch_ordered (CSR only, n < 2^31; a d_order with d_offsets == NULL is
 *           PIRE_GPU_EINVAL).
 *   Start   d_start: n device words, required for n > 0.  d_start[i] is a StateIndex in the reference's numbering and
 *           string i starts from it (with d_order too: every array is indexed by the original string number).  BEGIN
 *           steps BeginMark from each string's own start, END steps EndMark after its bytes.  A start >= Size() reads no
 *           table and yields match 0, mask 0 and state 0xFFFFFFFF, as in pire_gpu_run_string.
 *   Chain   the d_state_idx of a call made without END is the d_start of the next call, and it may be the same buffer:
 *           a batch of streams is updated in place round after round with no synchronise in between.
 *   flags   PIRE_GPU_RUN_BEGIN and/or PIRE_GPU_RUN_END; anything else (PIRE_GPU_RUN_LINES included) is PIRE_GPU_EINVAL,
 *           as are a NULL d_start and a NULL corpus with non-empty strings.  n == 0 is a no-op.
 *   Output  as pire_gpu_run_batch (bits past n are 0, nothing past n is written).
 * The kernel variant is chosen as pire_gpu_run_batch chooses it, AUTO's recorded choice included; PRIV runs PLAIN's
 * walk.  Asynchronous on `stream`; a host-only handle gets PIRE_GPU_ENODEVICE. */
int pire_gpu_run_batch_from(const pire_gpu_scanner* sc,
                            const uint8_t* d_corpus, const uint64_t* d_offsets, const uint32_t* d_order,
                            uint64_t fixed_len, uint64_t n, uint32_t flags,
                            const uint32_t* d_start,
                            uint32_t* d_match_bits, uint32_t* d_accept_masks, uint32_t* d_state_idx,
                            void* stream);

/* Two scanners over one batch.  Replaces, for every string i of a batch,
 *     Pire::Run(sc1, sc2, st1_i, st2_i, begin, end)                                        run.h:230-241
 *     Pire::Runner(Pire::ScannerPair(sc1, sc2)) [.Begin()] .Run(string i) [.End()]         scanners/pair.h
 * for a pattern set split over two scanners (Scanner::Glue stops at a size limit).  Each scanner's half of the result
 * is exactly what it gets alone on the same bytes: pire_gpu_run_batch_from(sc1, ..., d_start1, outputs 1) and the same
 * for sc2, or pire_gpu_run_batch when that scanner's start array is NULL.  ScannerPair's Final() is the OR of the two
 * match bits.
 *   Batch   as pire_gpu_run_batch: CSR (d_offsets) or fixed length; no order.
 *   flags   PIRE_GPU_RUN_BEGIN and/or PIRE_GPU_RUN_END, stepped for both scanners; anything else (PIRE_GPU_RUN_LINES
 *           included: the lines of a text have pire_gpu_run_pair_lines) is PIRE_GPU_EINVAL, as are a NULL corpus with
 *           non-empty strings and n > 2^40.
 *   Start   d_start1 / d_start2: n device words each, or NULL for Initialize().  A start >= Size() yields match 0, mask
 *           0 and state 0xFFFFFFFF for its own scanner only.
 *   Chain   d_state_idx1 may be d_start1 and d_state_idx2 may be d_start2: both halves of a batch of streams are updated
 *           in place round after round.  A buffer shared between the two scanners (d_state_idx2 == d_start1, say) is
 *           not supported.
 *   Output  as pire_gpu_run_batch, once per scanner; each of the six may be NULL.
 *   Handles both on one device (PIRE_GPU_EINVAL otherwise); a host-only handle gets PIRE_GPU_ENODEVICE.  sc1 may be
 *           sc2.  Each handle runs with its own hot set, tuned or not.
 * A uniform batch (fixed length a multiple of 32, corpus 32-byte aligned) is scanned in one pass: every byte is read
 * from HBM once and walked through both automata.  Any other batch is not fused: it runs as the two single-scanner
 * launches, one after the other on the stream.  n == 0 is a no-op.  Asynchronous on `stream`; re-entrant. */
int pire_gpu_run_pair_batch(const pire_gpu_scanner* sc1, const pire_gpu_scanner* sc2,
                            const uint8_t* d_corpus, const uint64_t* d_offsets, uint64_t fixed_len, uint64_t n,
                            uint32_t flags, const uint32_t* d_start1, const uint32_t* d_start2,
                            uint32_t* d_match_bits1, uint32_t* d_accept_masks1, uint32_t* d_state_idx1,
                            uint32_t* d_match_bits2, uint32_t* d_accept_masks2, uint32_t* d_state_idx2,
                            void* stream);

/* Replaces, per string of a batch,
 *     Pire::LongestPrefix(sc, begin, end, throughBeginMark, throughEndMark)   run.h:277-292
 *     Pire::ShortestPrefix(sc, begin, end, throughBeginMark, throughEndMark)   run.h:294-311
 * d_prefix_len[i] = length of the longest / shortest prefix of string i that the
 * scanner accepts, or PIRE_GPU_NO_PREFIX when there is none (the reference returns a
 * null pointer).  flags: PIRE_GPU_RUN_BEGIN = throughBeginMark, PIRE_GPU_RUN_END =
 * throughEndMark.  The scan stops in a dead state (pire_ut.cpp ScanTermination).
 * Semantics are those of the byte-by-byte predicates (run.h:69-100), i.e. of the
 * NoMask scanner variants: the ExitMasks fast-forward of the reference skips the
 * predicate for the bytes it jumps over, which can leave LongestPrefix short when a
 * string ends exactly on a 16-byte boundary of the host address space. */
#define PIRE_GPU_NO_PREFIX 0xFFFFFFFFu
int pire_gpu_prefix_batch(const pire_gpu_scanner* sc,
                          const uint8_t* d_corpus, const uint64_t* d_offsets,
                          uint64_t fixed_len, uint64_t n, uint32_t flags, int shortest,
                          uint32_t* d_prefix_len, void* stream);

/* Replaces, per string of a batch, the run of a Pire::HalfFinalScanner (pire/scanners/half_final.h):
 *     HalfFinalScanner::State st;  sc.Initialize(st);            half_final.h:136-141
 *     [Pire::Step(sc, st, BeginMark);]  Pire::Run(sc, st, begin, end);  [Pire::Step(sc, st, EndMark);]
 *     st.Result(r) for every regexp r                             half_final.h:88-90
 * (the driver of tests/count_ut.cpp:54-63).  TakeAction (half_final.h:154-163) adds one to the counter of
 * every regexp listed for a state each time the walk enters that state while it is final -- so Result(r)
 * counts the positions where a match of regexp r ends (HalfFinalFsm's counters, half_final_fsm.h:11-20),
 * and AcceptedRegexps(st) is { r : Result(r) != 0 }.
 * The image is the Save() stream of the HalfFinalScanner (it inherits Scanner::Save; the same format).
 * d_counts: n rows of max(1, regexps) u32, row i for string i (overwritten).  d_match_bits: packed
 * Final(st) per string, may be null.  Counters are 32 bits wide (the reference's are size_t). */
/* Replaces, per string of a batch,
 *     Pire::LongestSuffix (sc, rbegin, rend, throughEndMark, throughBeginMark)   run.h:316-342
 *     Pire::ShortestSuffix(sc, rbegin, rend, throughEndMark, throughBeginMark)   run.h:345-362
 * with rbegin = the string's last byte and rend = one before its first: the scanner (normally compiled from
 * Fsm::Reverse()) is walked over the string from right to left.  d_suffix_len[i] = length of the longest /
 * shortest suffix accepted that way (the reference returns the pointer rbegin - length), or
 * PIRE_GPU_NO_PREFIX for its null.  PIRE_GPU_RUN_END = throughEndMark (stepped before the bytes),
 * PIRE_GPU_RUN_BEGIN = throughBeginMark (stepped after them).  ShortestSuffix's quirk is kept: with
 * throughBeginMark the mark is stepped from the state the scan stopped in, and the answer is null unless that
 * state is final (run.h:357-360). */
int pire_gpu_suffix_batch(const pire_gpu_scanner* sc,
                          const uint8_t* d_corpus, const uint64_t* d_offsets,
                          uint64_t fixed_len, uint64_t n, uint32_t flags, int shortest,
                          uint32_t* d_suffix_len, void* stream);

/* How pire_gpu_count_batch keeps the counters (results are identical; for tests and measurements).
 * AUTO: packed per-state increments when the automaton has at most 16 regexps, behind a look-ahead pass
 * that skips chunks without final states -- or on every chunk when pire_gpu_scanner_tune saw more than
 * 2.5 % of the sample's steps end in a final state; the accept lists otherwise. */
#define PIRE_GPU_COUNT_AUTO        0u
#define PIRE_GPU_COUNT_LISTS       1u
#define PIRE_GPU_COUNT_PACKED      2u
#define PIRE_GPU_COUNT_EVERY_CHUNK 3u
int pire_gpu_scanner_set_count_mode(pire_gpu_scanner* sc, uint32_t mode);

int pire_gpu_count_batch(const pire_gpu_scanner* sc,
                         const uint8_t* d_corpus, const uint64_t* d_offsets,
                         uint64_t fixed_len, uint64_t n, uint32_t flags,
                         uint32_t* d_counts, uint32_t* d_match_bits, void* stream);

/* HalfFinalScanner counts of one long string with the whole GPU ("how many times does each pattern occur in this
 * file").  Replaces, for one string resident in HBM, the driver of tests/count_ut.cpp:54-63 with the state carried
 * across calls the way a HalfFinalScanner::State is:
 *     [sc.Initialize(st);]  [Pire::Step(sc, st, BeginMark);]  Pire::Run(sc, st, begin, end);  [Pire::Step(sc, st, EndMark);]
 * The string is cut into pieces and stitched as in pire_gpu_run_string, then every piece is counted from its true start.
 *   Input   d_text[0 .. n_bytes), any length (0 included; d_text may then be NULL), any alignment, past 4 GiB too.
 *   flags   PIRE_GPU_RUN_BEGIN steps BeginMark and counts the state it reaches; PIRE_GPU_RUN_END steps EndMark and
 *           counts the state it reaches.  Anything else is PIRE_GPU_EINVAL.
 *   Start   d_start == NULL: Initialize(), whose TakeAction is counted (half_final.h:136-141), as in
 *           pire_gpu_count_batch.  Otherwise d_start points to ONE device word holding a StateIndex in the reference's
 *           numbering; the run resumes from it and does NOT count it again (the call that reached it counted it).  A
 *           start >= Size() adds nothing and yields match 0 and state 0xFFFFFFFF, as in pire_gpu_run_string.
 *   Counts  d_counts (required): max(1, RegexpsCount()) u64 words that the call ADDS to -- unlike pire_gpu_count_batch,
 *           whose u32 rows are overwritten.  The caller zeroes them before the first call.  64 bits because one string
 *           can be longer than 2^32 bytes and a state can list a regexp more than once.
 *   Chain   the d_state_idx of a call made without END is the d_start of the next call, and it may be the same word;
 *           d_counts may be the same buffer.  A text arriving in chunks is counted with no synchronise in between
 *           (BEGIN on the first call, END on the last), and the result equals one call over the concatenated text.
 *   Output  each may be NULL: d_match_bits[0] = Final() of the last state (the whole word: bit 0, the others 0),
 *           d_state_idx[0] = its StateIndex (after End() with END).  Nothing else is written.
 * pire_gpu_scanner_set_count_mode is honoured; the results are identical in every mode.  Whenever the counts fit in 32
 * bits they equal pire_gpu_count_batch's with n = 1 (CSR) on the same bytes; match and state always equal
 * pire_gpu_run_string's.  A NULL d_counts and a NULL d_text with n_bytes > 0 are PIRE_GPU_EINVAL; a host-only handle
 * gets PIRE_GPU_ENODEVICE.  Asynchronous on `stream`; re-entrant across streams on one handle (per-call scratch).  It
 * costs about pire_gpu_run_string plus one more walk of the bytes, and shares its worst case (DESIGN.md 4). */
int pire_gpu_count_string(const pire_gpu_scanner* sc, const uint8_t* d_text, uint64_t n_bytes, uint32_t flags,
                          const uint32_t* d_start, uint64_t* d_counts,
                          uint32_t* d_match_bits, uint32_t* d_state_idx, void* stream);

/* Where the HalfFinalScanner matches end in one long string, with the whole GPU ("regexp 3 occurs 41 times in this log:
 * where?").  pire_gpu_count_string's run, listing every count it would add instead of adding it: each TakeAction
 * (half_final.h:154-163) yields one entry (end, id) for each id in the accept list of the state entered, in list order
 * (a state that lists an id twice yields two entries, as it adds two to the count).
 *   Input, flags, start and chain   exactly as in pire_gpu_count_string: BEGIN and/or END (anything else, LINES
 *           included, is PIRE_GPU_EINVAL); d_start == NULL is Initialize(), whose TakeAction is reported; a resumed
 *           start is not reported again; a start >= Size() reports nothing and yields match 0 and state 0xFFFFFFFF;
 *           d_state_idx may be d_start.
 *   end     base + the number of text bytes consumed when the state was entered: Initialize() and BeginMark are at
 *           base + 0, byte k of the text at base + k + 1, EndMark at base + n_bytes.
 *   Order   walk order: ascending end, and within one end in step order, then accept-list order.  The order is fully
 *           determined, so two calls on the same input write identical arrays.
 *   Output  *d_found (required) is one device u64 that the call reads and ADDS its number of entries to.  The call's
 *           k-th entry goes to index *d_found + k of d_ends (end) and d_ids (regexp id) if that index is < capacity;
 *           nothing at or past capacity and nothing below the incoming *d_found is written.  d_ends and d_ids may each
 *           be NULL (nothing goes to a NULL array).  With too small a buffer the written entries are exactly the first
 *           `capacity` entries of the full answer, and *d_found is still the full total, so the caller can tell and call
 *           again with a larger buffer.  d_match_bits[0] / d_state_idx[0] as in pire_gpu_count_string.
 *   Chain   zero *d_found once and pass the running byte offset as `base`: chained calls append, with no synchronise
 *           in between, and write what one call over the concatenated text writes.
 * The entries with id == r number exactly pire_gpu_count_string's Result(r) on the same bytes, flags and start; match
 * and state equal pire_gpu_run_string's.  pire_gpu_scanner_set_count_mode does not apply.  A NULL d_found and a NULL
 * d_text with n_bytes > 0 are PIRE_GPU_EINVAL; a host-only handle gets PIRE_GPU_ENODEVICE.  Asynchronous on `stream`;
 * re-entrant across streams on one handle (per-call scratch).  It costs about pire_gpu_count_string plus one more walk
 * of the bytes and the writes of the entries (DESIGN.md 4). */
int pire_gpu_match_ends_string(const pire_gpu_scanner* sc, const uint8_t* d_text, uint64_t n_bytes, uint32_t flags,
                               const uint32_t* d_start, uint64_t base,
                               uint64_t* d_ends, uint32_t* d_ids, uint64_t capacity, uint64_t* d_found,
                               uint32_t* d_match_bits, uint32_t* d_state_idx, void* stream);

/* HalfFinalScanner counts of many streams at once, each resumed from its own state ("how many times did each pattern
 * occur in each of these connections / log tails / files read block by block").  Replaces, for every string i of a
 * batch, the driver of tests/count_ut.cpp:54-63 with the state carried across calls the way a HalfFinalScanner::State is:
 *     [sc.Initialize(st_i);]  [Pire::Step(sc, st_i, BeginMark);]  Pire::Run(sc, st_i, begin_i, end_i);  [Pire::Step(sc, st_i, EndMark);]
 * One string per lane, on pire_gpu_count_batch's kernel.
 *   Batch   CSR or fixed length, as in pire_gpu_run_batch.  n == 0 is a no-op that writes nothing.
 *   flags   PIRE_GPU_RUN_BEGIN steps BeginMark from each string's own start and counts the state it reaches;
 *           PIRE_GPU_RUN_END steps EndMark after the string's bytes and counts the state it reaches.  Anything else
 *           (PIRE_GPU_RUN_LINES included) is PIRE_GPU_EINVAL.
 *   Start   d_start == NULL: every string starts from Initialize(), whose TakeAction is counted (half_final.h:136-141), as
 *           in pire_gpu_count_batch.  Otherwise d_start holds n StateIndex words in the reference's numbering; string i
 *           resumes from d_start[i] and does NOT count it again (the call that reached it counted it).  A start >= Size()
 *           reads no table and adds nothing; it yields match 0 and state 0xFFFFFFFF, and so stays in later rounds.  A
 *           stream that joins in a later round takes pire_gpu_initial()'s StateIndex as its start word; its Initialize()
 *           TakeAction is then not counted, which differs from a fresh start only when the initial state is final.
 *   Counts  d_counts (required): n rows of max(1, RegexpsCount()) u64 counters, row i for string i, that the call ADDS
 *           to -- like pire_gpu_count_string, unlike pire_gpu_count_batch, whose u32 rows are overwritten.  The caller
 *           zeroes them before the first call.  Nothing past row n - 1 is written.
 *   Chain   the d_state_idx of a call made without END is the d_start of the next call, and it may be the same buffer;
 *           d_counts is the same buffer in every round.  Rounds update one state array and one counter array in place
 *           with no synchronise in between, and the counts equal one call over each stream's concatenated pieces.  An
 *           empty string passes its state through unchanged (and still takes the marks the flags ask for).
 *   Output  each may be NULL: d_match_bits, Final() of each string's last state, packed (bits past n are 0);
 *           d_state_idx, n words, its StateIndex (after End() with END).
 * pire_gpu_scanner_set_count_mode is honoured; the results are identical in every mode.  With d_start == NULL and
 * zeroed counters the counts are pire_gpu_count_batch's, widened to u64, and so are the match bits; match bits and
 * states always equal pire_gpu_run_batch_from's on the same bytes and starts.  A NULL d_counts, a NULL corpus with
 * non-empty strings and n > 2^40 are PIRE_GPU_EINVAL; a host-only handle gets PIRE_GPU_ENODEVICE.  Asynchronous on
 * `stream`.  Not covered: ordered batches (d_order; the counting kernel has no length-binned launch) and line batches
 * (no per-string starts, as in pire_gpu_run_batch_from). */
int pire_gpu_count_batch_from(const pire_gpu_scanner* sc,
                              const uint8_t* d_corpus, const uint64_t* d_offsets,
                              uint64_t fixed_len, uint64_t n, uint32_t flags,
                              const uint32_t* d_start, uint64_t* d_counts,
                              uint32_t* d_match_bits, uint32_t* d_state_idx, void* stream);

/* Where the HalfFinalScanner matches end in many streams at once, each resumed from its own state ("regexp 3 occurred 41
 * times in stream 17: where?").  pire_gpu_count_batch_from's run, listing every count it would add instead of adding it:
 * each TakeAction of string i yields one entry (i, end, id) for each id in the accept list of the state entered, in list
 * order.  One string per lane, on pire_gpu_count_batch_from's kernel, in two walks around a scan of the strings' totals.
 *   Batch, flags, start and chain   exactly as in pire_gpu_count_batch_from: CSR or fixed length; BEGIN and/or END
 *           (anything else, LINES included, is PIRE_GPU_EINVAL); d_start == NULL is Initialize(), whose TakeAction is
 *           reported; a resumed start is not reported again; a start >= Size() reports nothing and yields match 0 and
 *           state 0xFFFFFFFF; d_state_idx may be d_start.
 *   Positions d_pos (n u64 words, or NULL: every base 0 and nothing written): d_pos[i] is the number of bytes stream i
 *           consumed before this call, the `base` of pire_gpu_match_ends_string.  Initialize() and BeginMark are at
 *           d_pos[i] + 0, byte k of string i at d_pos[i] + k + 1, EndMark at d_pos[i] + len_i.  The call adds len_i to
 *           d_pos[i] (also for an unknown start), so rounds chain with no host work.
 *   Order   by string index, then walk order within a string: ascending end, then step order, then accept-list order.
 *   Output  *d_found (required) is one device u64 that the call reads and ADDS its number of entries to.  The call's
 *           k-th entry goes to index *d_found + k of d_strings (string index), d_ends (end) and d_ids (regexp id) if that
 *           index is < capacity; nothing at or past capacity and nothing below the incoming *d_found is written.  Each of
 *           the three arrays may be NULL.  With too small a buffer the written entries are exactly the first `capacity`
 *           entries of the full answer, and *d_found is still the full total.  The placement comes from a scan, not from
 *           atomics: two calls on the same input write identical bytes.  d_match_bits / d_state_idx (each may be NULL)
 *           as in pire_gpu_count_batch_from.
 *   Chain   zero *d_found and d_pos once; the d_state_idx of a call made without END is the d_start of the next, and
 *           may be the same buffer.  Rounds append with no synchronise in between, and write what one call over each
 *           stream's concatenated pieces writes.
 * The entries of string i are what pire_gpu_match_ends_string writes for string i alone, with start d_start[i] (or
 * NULL) and base d_pos[i]; their per-id histogram is row i of pire_gpu_count_batch_from; match bits and states equal
 * pire_gpu_run_batch_from's.  pire_gpu_scanner_set_count_mode does not apply.  n == 0 is a no-op that writes nothing.  A
 * NULL d_found, a NULL corpus with non-empty strings and n >= 2^32 (string indices are u32) are PIRE_GPU_EINVAL; a
 * host-only handle gets PIRE_GPU_ENODEVICE.  Asynchronous on `stream`; re-entrant across streams on one handle (per-call
 * scratch).  It costs about pire_gpu_count_batch_from plus a walk of the strings that have entries, and the writes of the
 * entries (DESIGN.md 4).  Not covered, as in pire_gpu_count_batch_from: ordered batches (d_order) and line batches
 * (PIRE_GPU_RUN_LINES is refused; the lines of a text have pire_gpu_match_ends_lines). */
int pire_gpu_match_ends_batch_from(const pire_gpu_scanner* sc,
                                   const uint8_t* d_corpus, const uint64_t* d_offsets, uint64_t fixed_len, uint64_t n,
                                   uint32_t flags, const uint32_t* d_start, uint64_t* d_pos,
                                   uint32_t* d_strings, uint64_t* d_ends, uint32_t* d_ids, uint64_t capacity, uint64_t* d_found,
                                   uint32_t* d_match_bits, uint32_t* d_state_idx, void* stream);

/* Where the matches whose ends the two calls above list start: the span of each match, for grep -o, highlighting or
 * extracting a field.  Pire's own answer (run.h:312-342): LongestSuffix through a scanner built with Fsm::Reverse()
 * ("consider using Fsm::Reverse() for using in this function"), walked leftwards from the match's end.
 *   rsc     a plain Scanner image compiled from the same patterns with Fsm::Reverse() and without Surround(); for
 *           several regexps the reversed scanners glued in the order of the forward HalfFinalScanner, so that regexp
 *           ids agree.
 *   Window  the text bytes the caller still holds, numbered as the entries' ends.  String form: [base, base + n_bytes)
 *           of d_text.  Batch form (CSR or fixed length, as in pire_gpu_run_batch): string i covers
 *           [d_pos[i] - len_i, d_pos[i]), d_pos being match_ends_batch_from's array as that call leaves it (one past
 *           each string's last byte), so the same buffer is passed straight on; d_pos == NULL means len_i (ends are
 *           offsets within each string).  d_strings == NULL means every entry belongs to string 0.
 *   Entries indices [*d_first, min(*d_found, capacity)) of d_strings / d_ends / d_ids, as match_ends wrote them.  Both
 *           words are read on the device, so this call can follow a match-ends call on the same stream with no
 *           synchronise; d_first == NULL means 0.  A caller that chains chunks copies *d_found into d_first (8 bytes,
 *           device to device) before each match-ends call.  An entry whose end lies outside its string's window, or
 *           whose string is >= n, is not written: one entry array can be processed window by window.
 *   Answer  d_starts[k]: the least s such that the reversed walk from end_k leftwards accepts over [s, end_k), where
 *           "accepts" means id_k is in AcceptedRegexps(state) -- Final(state) when d_ids == NULL, which is exactly
 *           LongestSuffix -- or PIRE_GPU_NO_START.  The walk steps BeginMark last when it reaches the window start and
 *           PIRE_GPU_RUN_BEGIN says that is where the text begins.  An entry at the window's end under PIRE_GPU_RUN_END
 *           is walked twice, without and with EndMark stepped first, and the longer answer is kept (a match-ends entry
 *           does not record whether its match took the EndMark step); every other entry is walked without EndMark.  So
 *           start_k is the leftmost start of a match of id_k ending at end_k, with BeginMark and EndMark only at the
 *           text's real edges.  max_back > 0 bounds each walk to [max(window start, end_k - max_back), end_k); BeginMark
 *           is then stepped only when that bound is the window start.
 *   Open    d_open[k] (may be NULL) is 1 when a walk of entry k reached its lower bound in a state from which id_k
 *           (with d_ids == NULL: a final state) can still be accepted and no BeginMark step settled it: bytes further
 *           left could move the start left, so the caller may widen the window (or max_back) and call again.
 *   flags   PIRE_GPU_RUN_BEGIN and/or PIRE_GPU_RUN_END; anything else (LINES included) is PIRE_GPU_EINVAL.  The
 *           entries of pire_gpu_match_ends_lines have pire_gpu_match_starts_lines.
 * Nothing outside the processed index range is written.  A NULL d_ends, d_found or d_starts and a NULL text with a
 * non-empty window are PIRE_GPU_EINVAL; a host-only handle gets PIRE_GPU_ENODEVICE; n == 0 or capacity == 0 is a
 * no-op.  Asynchronous on `stream`; re-entrant across streams on one handle (per-call scratch).  One entry per lane,
 * each walk stopped as soon as id_k can no longer be accepted.  Worst case: a reversed regexp that never dies (the forward
 * pattern has a .*-like prefix, e.g. hello\s+w.+d$ over printable text) walks back to the lower bound for every such
 * entry, serially, at the speed of one lane; max_back is the bound for that case (DESIGN.md 4). */
#define PIRE_GPU_NO_START 0xFFFFFFFFFFFFFFFFull
int pire_gpu_match_starts_string(const pire_gpu_scanner* rsc, const uint8_t* d_text, uint64_t n_bytes, uint64_t base,
                                 uint32_t flags, uint64_t max_back,
                                 const uint64_t* d_ends, const uint32_t* d_ids,
                                 const uint64_t* d_first, const uint64_t* d_found, uint64_t capacity,
                                 uint64_t* d_starts, uint8_t* d_open, void* stream);
int pire_gpu_match_starts_batch(const pire_gpu_scanner* rsc, const uint8_t* d_corpus, const uint64_t* d_offsets,
                                uint64_t fixed_len, uint64_t n, const uint64_t* d_pos, uint32_t flags, uint64_t max_back,
                                const uint32_t* d_strings, const uint64_t* d_ends, const uint32_t* d_ids,
                                const uint64_t* d_first, const uint64_t* d_found, uint64_t capacity,
                                uint64_t* d_starts, uint8_t* d_open, void* stream);

/* The step before the path for line-oriented input (samples/pigrep/pigrep.cpp:38-45 calls
 * std::getline and then Runner(sc).Begin().Run(line).End() per line).
 * pire_gpu_split_lines finds the lines of a newline-delimited text resident in HBM:
 *   d_line_offsets[0..*n_lines] (capacity + 1 entries available), line i =
 *   d_text[off[i] .. off[i+1] - 1) -- the newline itself is excluded, a last line without
 *   newline is kept, an empty text has no lines (std::getline semantics).
 *   If capacity is too small (or d_line_offsets is NULL) nothing is written, *n_lines
 *   receives a sufficient capacity and PIRE_GPU_EINVAL is returned.  Synchronises `stream`.
 * pire_gpu_run_lines scans those lines; outputs as in pire_gpu_run_batch.  d_line_offsets must be the offsets
 *   pire_gpu_split_lines produced for d_text: without d_order the lines are scanned where they lie -- every lane
 *   walks a few KiB of the text and restarts behind each newline it meets -- so line i + 1 has to start right behind the
 *   newline that ends line i.  With d_order (pire_gpu_length_order; usually slower for lines) they are scanned one
 *   string per lane like any CSR batch. */
int pire_gpu_split_lines(const uint8_t* d_text, uint64_t n_bytes, uint64_t* d_line_offsets, uint64_t capacity,
                         uint64_t* n_lines, int device, void* stream);
int pire_gpu_run_lines(const pire_gpu_scanner* sc, const uint8_t* d_text, const uint64_t* d_line_offsets,
                       const uint32_t* d_order, uint64_t n_lines, uint32_t flags,
                       uint32_t* d_match_bits, uint32_t* d_accept_masks, uint32_t* d_state_idx, void* stream);

/* Two scanners over the lines of a text.  Replaces, for every line of the text,
 *     Pire::Runner(Pire::ScannerPair(sc1, sc2)) [.Begin()] .Run(line) [.End()]            scanners/pair.h
 * for a pattern set split over two scanners, as pigrep with two scanners runs it.  Each scanner's three outputs are,
 * bit for bit, what pire_gpu_run_lines(sc_k, d_text, d_line_offsets, NULL, n_lines, flags, ...) writes, the zeroed bits
 * past n_lines in the last bitmap word included.  ScannerPair's Final() is the OR of the two match bits.
 *   Lines   d_line_offsets are the offsets pire_gpu_split_lines made for d_text, as pire_gpu_run_lines requires.  Every
 *           line starts from Initialize(); there is no order and no start state.
 *   flags   PIRE_GPU_RUN_BEGIN and/or PIRE_GPU_RUN_END, stepped for both scanners; PIRE_GPU_RUN_LINES is implied and
 *           accepted; anything else is PIRE_GPU_EINVAL, as are a NULL text or offsets with lines and n_lines >= 2^31.
 *   Output  as pire_gpu_run_lines, once per scanner; each of the six may be NULL.  A buffer shared between the two
 *           scanners' outputs is not supported.
 *   Handles both on one device (PIRE_GPU_EINVAL otherwise); a host-only handle gets PIRE_GPU_ENODEVICE.  sc1 may be
 *           sc2.  Each handle runs with its own hot set, tuned or not.
 * When both start states are hot rows (practically always) the text is walked once: every byte is read from HBM once and
 * walked through both automata.  Otherwise each scanner runs its own pire_gpu_run_lines launch, one after the other on
 * the stream.  n_lines == 0 is a no-op.  Asynchronous on `stream`; re-entrant. */
int pire_gpu_run_pair_lines(const pire_gpu_scanner* sc1, const pire_gpu_scanner* sc2,
                            const uint8_t* d_text, const uint64_t* d_line_offsets, uint64_t n_lines, uint32_t flags,
                            uint32_t* d_match_bits1, uint32_t* d_accept_masks1, uint32_t* d_state_idx1,
                            uint32_t* d_match_bits2, uint32_t* d_accept_masks2, uint32_t* d_state_idx2,
                            void* stream);

/* Where the HalfFinalScanner matches end in every line of a text (grep -o, grep -n, grep -b): each line is its own run,
 * Runner(sc).Begin().Run(line).End() as samples/pigrep runs it, listed as pire_gpu_match_ends_batch_from lists a batch.
 *   Lines   d_line_offsets are the offsets pire_gpu_split_lines made for d_text, as pire_gpu_run_lines requires; line l
 *           is d_text[off[l], off[l+1] - 1).
 *   Run     every line from Initialize(), whose TakeAction is reported; with BEGIN, BeginMark is stepped and reported;
 *           then the line's bytes; with END, EndMark is stepped and reported.  Each TakeAction yields one entry (l, end,
 *           id) for each id in the accept list of the state entered, in list order.
 *   Positions are the text's: Initialize() and BeginMark at off[l], byte k of line l at off[l] + k + 1, EndMark at
 *           off[l+1] - 1.  So the entries index d_text directly, and pire_gpu_match_starts_lines takes them as they are.
 *   Order   ascending line, then walk order within a line.  The placement comes from a scan, not from atomics: two calls
 *           on the same input write identical bytes.
 *   Output  as in pire_gpu_match_ends_batch_from: *d_found (required) is read and ADDED to; the call's k-th entry goes to
 *           index *d_found + k of d_lines, d_ends and d_ids (each may be NULL) if that index is < capacity, and a short
 *           buffer holds exactly the first `capacity` entries of the full answer while *d_found is still the full total.
 *           d_match_bits / d_state_idx (each may be NULL) are what pire_gpu_run_lines gives with the same handle and
 *           flags; bits past n_lines are 0.
 *   flags   PIRE_GPU_RUN_BEGIN and/or PIRE_GPU_RUN_END; PIRE_GPU_RUN_LINES is implied and accepted; anything else is
 *           PIRE_GPU_EINVAL.
 * The entries of line l are exactly what pire_gpu_match_ends_string writes for that line alone (d_start NULL, the same
 * flags, base off[l]); their per-id histogram is row l of pire_gpu_count_batch with PIRE_GPU_RUN_LINES.  A NULL d_found,
 * NULL offsets, a NULL text with lines and n_lines >= 2^32 (line indices are u32) are PIRE_GPU_EINVAL; a host-only handle
 * gets PIRE_GPU_ENODEVICE; n_lines == 0 is a no-op.  Asynchronous on `stream`; re-entrant across streams on one handle
 * (per-call scratch).  The lines are walked where they lie, as in pire_gpu_run_lines, in two walks around a scan
 * (DESIGN.md 4); a handle whose start state is not a hot row walks one line per lane.  Not covered: resuming lines
 * across calls and ordered line batches.
 *
 * pire_gpu_match_starts_lines: pire_gpu_match_starts_batch for those entries, with each entry's window its own line
 * [off[l], off[l+1] - 1) and its end and start positions of the text.  BEGIN steps BeginMark at each line's start; END
 * walks an entry at its line's end with and without EndMark; max_back, d_open, d_first and the window rules (entries
 * outside their line, or with l >= n_lines, are not written) are unchanged.  The answer for entry k is that of
 * pire_gpu_match_starts_string with line l as its window and base off[l].  d_lines and the offsets are required
 * (PIRE_GPU_EINVAL without them); PIRE_GPU_RUN_LINES is accepted. */
int pire_gpu_match_ends_lines(const pire_gpu_scanner* sc, const uint8_t* d_text, const uint64_t* d_line_offsets,
                              uint64_t n_lines, uint32_t flags,
                              uint32_t* d_lines, uint64_t* d_ends, uint32_t* d_ids, uint64_t capacity, uint64_t* d_found,
                              uint32_t* d_match_bits, uint32_t* d_state_idx, void* stream);
int pire_gpu_match_starts_lines(const pire_gpu_scanner* rsc, const uint8_t* d_text, const uint64_t* d_line_offsets,
                                uint64_t n_lines, uint32_t flags, uint64_t max_back,
                                const uint32_t* d_lines, const uint64_t* d_ends, const uint32_t* d_ids,
                                const uint64_t* d_first, const uint64_t* d_found, uint64_t capacity,
                                uint64_t* d_starts, uint8_t* d_open, void* stream);

/* Same call with HOST buffers -- what a Pire user holds: Run(const char* begin, const char* end) takes pageable
 * memory (run.h:271-275; samples/pigrep/pigrep.cpp:38-45).  The corpus is cut into chunks of whole 32-string
 * units (about 64 MiB; PIRE_B200_HOST_CHUNK_MB) and streamed through a ring of three device slots: the
 * host->device copy of chunk k+1 overlaps the scan of chunk k and the device->host copy of its results.
 * Pageable input is staged through the library's own pinned buffers by a few copy threads
 * (PIRE_B200_HOST_THREADS, default min(8, cores / 4)); pinned or cudaHostRegister-ed input is DMA-ed straight
 * from the caller's buffer.  The device never holds more than the ring, so corpora larger than HBM stream through.
 * CSR batches are length-binned per chunk (pire_gpu_length_order).  Results are those of pire_gpu_run_batch on
 * the resident corpus.  Returns after everything has landed in the caller's arrays.
 * corpus_bytes = size of the corpus buffer; offsets (if any) must ascend and end within it, n * fixed_len
 * must fit in it (PIRE_GPU_EINVAL otherwise).  A line batch (PIRE_GPU_RUN_LINES, the offsets of
 * pire_gpu_split_lines for the text) needs the text up to offsets[n] - 1 only: a last line without '\n' has its
 * separator one byte past the text, so corpus_bytes = the text's size is right with or without a final newline.
 * Line batches are not length-binned; lines are scanned where they lie, as in pire_gpu_run_lines.
 * Concurrency: calls on one handle from several threads run concurrently, each with its own workspace
 * (streams, slots, staging); workspaces are kept with the handle and freed by pire_gpu_scanner_destroy. */
int pire_gpu_run_batch_host(const pire_gpu_scanner* sc,
                            const uint8_t* corpus, uint64_t corpus_bytes, const uint64_t* offsets,
                            uint64_t fixed_len, uint64_t n, uint32_t flags,
                            uint32_t* match_bits, uint32_t* accept_masks, uint32_t* state_idx);

/* A text of any size, from host memory, as device frames of whole lines (std::getline's loop of
 * samples/pigrep/pigrep.cpp:15-21 over a stream that never has to fit in HBM).  The caller hands over the text's
 * bytes in pieces of any size, split anywhere (read() blocks, an mmap'd file, a pinned buffer); every feed copies
 * as many of them as fit into the next of three device slots, behind the line carried over from the slot before,
 * and returns one frame: the slot's complete lines with the offsets pire_gpu_split_lines makes for them.
 *   Feeding  *consumed receives the number of bytes taken from `bytes`; the caller calls again with the rest.  A
 *            frame may have n_lines == 0 (no newline has arrived yet; its first offset word is 0).  With `last` set
 *            and every byte consumed, the open line becomes the text's last line (no newline, as split_lines keeps
 *            it) and the stream is finished: a later feed is PIRE_GPU_EINVAL.  An empty text has no lines; a text
 *            ending in '\n' has no extra empty line.
 *   Frames   lines are split_lines' lines of the whole text.  Shift a frame's offsets by first_byte and its line
 *            numbers by first_line: the frames in order give split_lines over the concatenated text word for word
 *            (frame k's last offset is frame k + 1's first one).  So a frame is accepted as it is by every call that
 *            takes split_lines offsets: pire_gpu_run_lines, pire_gpu_count_batch with PIRE_GPU_RUN_LINES,
 *            pire_gpu_match_ends_lines and pire_gpu_match_starts_lines.  The bytes behind a frame's last '\n' are
 *            carried to the head of the next slot by a device-to-device copy, never sent again from the host.
 *   Long lines  a line that does not fit in a slot grows the slot (at least doubling the room, so a long line is
 *            copied device-to-device O(1) times per byte); only a line larger than free device memory fails
 *            (PIRE_GPU_ECUDA with the CUDA message).  slot_bytes == 0 picks 256 MiB, the fastest of 16, 64 and 256 MiB
 *            in tools/line_stream_bench.py (DESIGN.md 4); the device then holds about 0.8 GiB of slots and offsets.
 *   Ordering  the bytes are copied and the lines found on the stream object's own stream, so the copy of frame
 *            k + 1 overlaps the caller's work on frame k.  Everything a frame needs is in place for work the caller
 *            enqueues on `stream` after feed returns.  The slot of frame k is written again by the feed that makes
 *            frame k + 3; before writing it, that feed orders itself after the work that was enqueued on `stream`
 *            when the feed making frame k + 1 was called.  So: work on frame k must be enqueued before the next feed
 *            is called (on the `stream` passed to that feed), and the frame's buffers stay valid until it completes.
 *            feed blocks until its own copies and the line split are done (split_lines synchronises) and until
 *            the work on frame k - 3's slot has finished; it never waits for the work on frame k - 1.  When feed
 *            returns, the caller's `bytes` are no longer referenced.
 *   Input    pageable bytes are staged through the library's pinned buffers by its copy threads
 *            (PIRE_B200_HOST_THREADS), pinned or cudaHostRegister-ed bytes are DMA-ed from the caller's buffer.
 *   Errors   NULL bytes with n > 0, a NULL consumed or frame are PIRE_GPU_EINVAL; device < 0 or a device that does
 *            not exist is PIRE_GPU_ENODEVICE at create.  A stream object belongs to one thread at a time.
 * pire_gpu_line_stream_destroy synchronises the device (the caller's work on the last frames reads the slots) and
 * frees the slots. */
typedef struct pire_gpu_line_stream pire_gpu_line_stream;
typedef struct pire_gpu_line_frame {
    const uint8_t* d_text;            /* the frame's bytes on the device                                           */
    const uint64_t* d_line_offsets;   /* n_lines + 1 words: what pire_gpu_split_lines makes for d_text, n_bytes    */
    uint64_t n_lines;
    uint64_t n_bytes;                 /* bytes of d_text (split_lines' n_bytes)                                    */
    uint64_t first_line;              /* index in the whole text of the frame's line 0                             */
    uint64_t first_byte;              /* offset in the whole text of d_text[0]                                     */
} pire_gpu_line_frame;
int pire_gpu_line_stream_create(int device, uint64_t slot_bytes, pire_gpu_line_stream** out);
int pire_gpu_line_stream_feed(pire_gpu_line_stream* ls, const uint8_t* bytes, uint64_t n, int last, void* stream,
                              uint64_t* consumed, pire_gpu_line_frame* frame);
void pire_gpu_line_stream_destroy(pire_gpu_line_stream* ls);

/* ---- several GPUs of one box ---------------------------------------------------
 * The path shards by string (SURVEY.md 8(e)): rank r of `world` scans the contiguous shard
 * pire_gpu_shard_bounds(n_global, world, r) -- boundaries on multiples of 32 strings, so bitmap words never straddle
 * ranks -- straight into its slot of the full-length match bitmap, and one in-place ncclAllGather of the equal-sized
 * slots completes the bitmap on every rank (1/world of the bytes of an all-reduce of a zeroed bitmap and no zeroing;
 * the shards are disjoint and word aligned, so the result is the same OR).  The reference's callers are C++
 * (tools/bench/bench.cpp:241-254, samples/pigrep/pigrep.cpp:38-45): this is their multi-GPU entry, no Python or
 * PyTorch involved.  NCCL is bound at run time (libnccl.so.2 of the process, else the system's); single-GPU users carry
 * no NCCL dependency, and these calls return PIRE_GPU_EUNSUPPORTED where NCCL is absent.
 *
 * One communicator per rank (process or thread; one GPU each):
 *   rank 0: pire_gpu_comm_get_id(id)  -> ship the PIRE_GPU_COMM_ID_BYTES bytes to every rank by any means
 *   every rank: pire_gpu_comm_create(id, world, rank, device, &comm)      (collective, like ncclCommInitRank)
 *   or pire_gpu_comm_adopt(ncclComm_t, device, &comm) around a communicator the caller already owns.
 * pire_gpu_run_sharded: d_corpus / d_offsets / d_accept_masks / d_state_idx describe THIS RANK's shard only (string
 *   0 of the buffers is string lo of the batch); d_match_bits_all has pire_gpu_sharded_words(n_global, world) words
 *   (>= ceil(n_global / 32); bits past n_global are zero) and is identical on every rank afterwards.  The scan runs
 *   on `stream`, the exchange on the communicator's own stream behind it.  Default: `stream` then waits for the
 *   exchange (stream-ordered, like any other call).  With PIRE_GPU_RUN_ASYNC_EXCHANGE the exchange is left running so
 *   that the caller's next work on `stream` (the next batch's scan into ANOTHER bitmap buffer) overlaps it;
 *   pire_gpu_comm_wait(comm, stream) makes `stream` wait for the last exchange before the bitmap is read.
 *   A later run_sharded on the same communicator orders itself after the pending exchange. */
#define PIRE_GPU_COMM_ID_BYTES 128
#define PIRE_GPU_RUN_ASYNC_EXCHANGE 8u
typedef struct pire_gpu_comm pire_gpu_comm;
void     pire_gpu_shard_bounds(uint64_t n_global, int world, int rank, uint64_t* lo, uint64_t* hi);
uint64_t pire_gpu_sharded_words(uint64_t n_global, int world);
int  pire_gpu_comm_get_id(void* id_out);
int  pire_gpu_comm_create(const void* id, int world, int rank, int device, pire_gpu_comm** out);
int  pire_gpu_comm_adopt(void* nccl_comm, int device, pire_gpu_comm** out);
void pire_gpu_comm_destroy(pire_gpu_comm* comm);
int  pire_gpu_comm_info(const pire_gpu_comm* comm, int* world, int* rank);
int  pire_gpu_comm_wait(pire_gpu_comm* comm, void* stream);
/* the exchange alone, for a slot filled some other way (e.g. uploaded after pire_gpu_run_batch_host); flags: 0 or
 * PIRE_GPU_RUN_ASYNC_EXCHANGE */
int  pire_gpu_comm_gather_bits(pire_gpu_comm* comm, uint64_t n_global, uint32_t* d_match_bits_all, uint32_t flags, void* stream);
int  pire_gpu_run_sharded(const pire_gpu_scanner* sc, pire_gpu_comm* comm,
                          const uint8_t* d_corpus, const uint64_t* d_offsets, uint64_t fixed_len,
                          uint64_t n_global, uint32_t flags,
                          uint32_t* d_match_bits_all, uint32_t* d_accept_masks, uint32_t* d_state_idx, void* stream);

/* Re-selects the shared-memory hot rows from the states a device-resident
 * sample of the workload actually visits (the reference has no counterpart; it
 * relies on the CPU cache to keep hot rows close).  Only speed depends on it.
 * Synchronises the device.  Not thread-safe against concurrent runs. */
int pire_gpu_scanner_tune(pire_gpu_scanner* sc,
                          const uint8_t* d_corpus, const uint64_t* d_offsets,
                          uint64_t fixed_len, uint64_t n_sample, uint32_t flags, void* stream);

/* Times every kernel variant that can serve this batch shape (two launches each,
 * results discarded) and makes the fastest one the handle's AUTO choice for that
 * shape (fixed-length/aligned vs generic).  ms_out[PIRE_GPU_VARIANT_SLOTS] (may be NULL) receives the
 * milliseconds per variant id, 0 for variants that do not apply.  Which variant
 * wins depends on the automaton and the text (see DESIGN.md section 4), so it is
 * measured rather than guessed.  Synchronises the device. */
int pire_gpu_scanner_autoselect(pire_gpu_scanner* sc,
                                const uint8_t* d_corpus, const uint64_t* d_offsets,
                                uint64_t fixed_len, uint64_t n, uint32_t flags, void* stream, float* ms_out);

/* AcceptedRegexps for scanners with MORE than 32 regexps (multi.h:149-158 returns a list of any length; Glue only
 * caps the states, multi.h:1092-1103).  The scan entry points' d_accept_masks holds ids 0..31; the complete answer
 * comes from the state each string stopped in: run with d_state_idx, then
 *     pire_gpu_accept_sets(sc, d_state_idx, n, d_sets, stream)
 * writes n rows of pire_gpu_accept_words(sc) = ceil(max(1, RegexpsCount()) / 32) words, bit (r % 32) of word
 * r / 32 of row i set iff regexp r is in AcceptedRegexps of string i's last state (after End() when the run
 * stepped it).  A state index outside the scanner yields an empty set. */
uint32_t pire_gpu_accept_words(const pire_gpu_scanner* sc);
int pire_gpu_accept_sets(const pire_gpu_scanner* sc, const uint32_t* d_state_idx, uint64_t n,
                         uint32_t* d_accept_sets, void* stream);

/* Number of kernels this library has launched in the calling process. */
uint64_t pire_gpu_launch_count(void);

/* ---- host-side Scanner concept on the flattened tables ------------------------
 * Index-space mirror of the concept the templates in run.h consume
 * (multi.h:137-194,:281-284); used by include/pire_gpu.hpp's HostScanner and by
 * the parity tests.  States are StateIndex values of the reference. */
uint32_t pire_gpu_initial(const pire_gpu_scanner* sc);                                   /* Initialize  multi.h:161 */
uint32_t pire_gpu_next(const pire_gpu_scanner* sc, uint32_t state, uint32_t ch);         /* Next        multi.h:189-192; ch in 0..259 */
int      pire_gpu_final(const pire_gpu_scanner* sc, uint32_t state);                     /* Final       multi.h:143 */
int      pire_gpu_dead(const pire_gpu_scanner* sc, uint32_t state);                      /* Dead        multi.h:147 */
size_t   pire_gpu_accepted_regexps(const pire_gpu_scanner* sc, uint32_t state,
                                   uint32_t* ids, size_t cap);                           /* AcceptedRegexps multi.h:149-158 */

/* ---- Pire::SlowScanner: patterns that cannot be determinised ---------------------
 * Replaces, for every string i of a batch,
 *     Pire::Runner(sc[, st_i]) [.Begin()] .Run(string i) [.End()]                          run.h:365-392
 * on a Pire::SlowScanner (slow.h:43-50), the scanner Pire::Regexp falls back to when Fsm::Determine() fails
 * (easy.h:205-215): x.{40}$, foo.{64}bar, approximate matching.  Its state is a SET of NFA states; here a set is W =
 * ceil(Size() / 32) u32 words, bit s of word s / 32 = state s in the reference's numbering (SlowScanner::State's flags).
 *   Create  `image` is the SlowScanner::Save() stream (header type 3; scanner_io.cpp:71-110).  Rejected with
 *           PIRE_GPU_EIMAGE: what SlowScanner::Load / Mmap reject, and a start, jump or letter outside the automaton, jump
 *           positions that step back or past the image, no states or no letters.  More than 4096 states is
 *           PIRE_GPU_EUNSUPPORTED.  An image of SlowScanner::Null() (Empty(), slow.h:427-431) has one state and never
 *           matches.  device == -1 builds a host-only handle (the host concept below; runs get PIRE_GPU_ENODEVICE).
 *           pire_gpu_scanner_create refuses SlowScanner images, as before.
 *   Batch   as pire_gpu_run_batch: CSR (d_offsets) or fixed length; with PIRE_GPU_RUN_LINES the offsets come from
 *           pire_gpu_split_lines and string i ends one byte before offsets[i+1].
 *   Start   d_start_sets NULL: Initialize() = {start}.  Otherwise n rows of W words; string i starts from row i
 *           (Runner(sc, st_i)); bits at or past Size() in a row are ignored.  BEGIN steps BeginMark from each start.
 *   Chain   d_sets may be d_start_sets: a batch of streams is carried on in place round after round, no synchronise.
 *   Output  each may be NULL.  d_match_bits: ceil(n/32) words, bit (i%32) of word i/32 = Final() (slow.h:152-158), bits
 *           past n are 0.  AcceptedRegexps() is {0} exactly when the bit is set (slow.h:165-167).  d_sets: n rows of W
 *           words, the set after End() (after the bytes without END), bits past Size() 0.
 *   flags   PIRE_GPU_RUN_BEGIN, PIRE_GPU_RUN_END, PIRE_GPU_RUN_LINES; anything else is PIRE_GPU_EINVAL, as are LINES with
 *           start sets or without offsets, a NULL corpus with non-empty strings and n > 2^40.  n == 0 is a no-op.
 * Scanners of at most 256 states walk one string per lane, larger ones one string per warp (DESIGN.md 4).  The walk of a
 * string stops early when its set is empty (nothing can match any more); the results are what End() would give.
 * Asynchronous on `stream`; re-entrant across streams on one handle. */
typedef struct pire_gpu_slow_scanner pire_gpu_slow_scanner;

typedef struct pire_gpu_slow_info {
    uint32_t states;           /* SlowScanner::Size()             slow.h:83 */
    uint32_t letters;          /* SlowScanner::GetLettersCount()  slow.h:81 */
    uint32_t regexps;          /* RegexpsCount(): 0 when Empty(), else 1  slow.h:88 */
    uint32_t set_words;        /* W = ceil(states / 32) */
    uint32_t start;            /* Initialize()'s one state */
    uint32_t empty;            /* Empty() */
    uint64_t table_bytes;      /* device bytes of the successor rows */
    uint64_t shared_bytes;     /* rows staged into shared memory per CTA (0: read through L1/L2) */
    int32_t  device;           /* CUDA device, or -1 for a host-only handle */
    uint32_t reserved;
} pire_gpu_slow_info;

int  pire_gpu_slow_scanner_create(const void* image, size_t size, int device, pire_gpu_slow_scanner** out);
void pire_gpu_slow_scanner_destroy(pire_gpu_slow_scanner* sc);
int  pire_gpu_slow_scanner_info(const pire_gpu_slow_scanner* sc, pire_gpu_slow_info* out);
int  pire_gpu_slow_run_batch(const pire_gpu_slow_scanner* sc,
                             const uint8_t* d_corpus, const uint64_t* d_offsets, uint64_t fixed_len, uint64_t n,
                             uint32_t flags, const uint32_t* d_start_sets,
                             uint32_t* d_match_bits, uint32_t* d_sets, void* stream);
/* Host-side concept on the parsed tables, sets of W words (bits past Size() in an input are ignored). */
int  pire_gpu_slow_initial(const pire_gpu_slow_scanner* sc, uint32_t* set);                  /* Initialize slow.h:91-97 */
int  pire_gpu_slow_next(const pire_gpu_slow_scanner* sc, const uint32_t* set, uint32_t ch,
                        uint32_t* out);                                                       /* Next slow.h:132-135; ch 0..259 */
int  pire_gpu_slow_final(const pire_gpu_slow_scanner* sc, const uint32_t* set);             /* Final slow.h:152-158: 1 or 0 */

/* ---- deterministic synthetic corpora (bench + tests) ---------------------------
 * Counter-based generator, identical bytes on host and device (SURVEY.md 8(d)).
 * kind 0: printable ASCII 0x20..0x7E; every `plant_every`-th string carries one
 *         planted literal, plants[(i / plant_every) % n_plants].  A literal
 *         starting with '^' is placed at the start of the string, one starting
 *         with '$' at its end (for anchored patterns; the marker itself is not
 *         written), any other at a pseudo-random offset, and then the string's
 *         last byte is set to `tail` when tail != 0.
 * `plants` is n_plants NUL-terminated literals back to back (plants_bytes in all). */
typedef struct pire_gpu_synth {
    uint64_t seed;
    uint64_t first_string;     /* global index of string 0 of this buffer (sharding) */
    uint64_t n_strings;
    uint32_t string_len;       /* fixed length, multiple of 16 */
    uint32_t kind;
    uint32_t plant_every;      /* 0 = never */
    uint32_t n_plants;
    const char* plants;
    uint32_t plants_bytes;
    uint32_t tail;
} pire_gpu_synth;

int pire_gpu_synth_fill_device(const pire_gpu_synth* spec, uint8_t* d_corpus, int device, void* stream);
int pire_gpu_synth_fill_host(const pire_gpu_synth* spec, uint8_t* corpus, uint64_t first, uint64_t count);
/* strings indices[0..count) of the corpus (relative to spec->first_string), back to back: stratified parity samples */
int pire_gpu_synth_fill_host_indexed(const pire_gpu_synth* spec, uint8_t* corpus, const uint64_t* indices, uint64_t count);

/* kind 1: mixed-length UTF-8 corpus (BASELINE config 4): lengths log-uniform in
 * [16, 65536), multiples of 4; ASCII / 2-byte Cyrillic / 3-byte code points; every
 * plant_every-th string (>= 32 bytes) ends with a mixed-case hit for the
 * case-insensitive headline pattern.  *_lengths_* writes n lengths (the caller
 * prefix-sums them into CSR offsets); *_fill_* writes the bytes for given offsets. */
int pire_gpu_synth_mixed_lengths_device(uint64_t seed, uint64_t first_string, uint64_t n, uint64_t* d_lengths, int device, void* stream);
int pire_gpu_synth_mixed_lengths_host(uint64_t seed, uint64_t first_string, uint64_t n, uint64_t* lengths);
int pire_gpu_synth_mixed_fill_device(uint64_t seed, uint32_t plant_every, uint64_t first_string, uint64_t n,
                                     const uint64_t* d_offsets, uint8_t* d_corpus, int device, void* stream);
int pire_gpu_synth_mixed_fill_host(uint64_t seed, uint32_t plant_every, uint64_t first_string, uint64_t n,
                                   const uint64_t* offsets, uint8_t* corpus);

const char* pire_gpu_last_error(void);
const char* pire_gpu_version(void);

#ifdef __cplusplus
}
#endif
#endif
