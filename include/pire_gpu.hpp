// pire_gpu.hpp -- header-only C++ mirror of Pire's Scanner / Runner / Matches
// surface over the C ABI of include/pire_b200.h.
//
// For a code base that already uses Pire:
//
//     Pire::Scanner sc = Pire::Lexer("hello\\s+w.+d$").Parse().Surround().Compile<Pire::Scanner>();
//     Pire::Gpu::Scanner gsc(sc, /*device*/ 0);              // Scanner::Save() -> device tables
//     Pire::Gpu::Batch batch{d_corpus, d_offsets, 0, n};     // strings resident in HBM
//     Pire::Gpu::BatchRunner r = Pire::Gpu::Runner(gsc);
//     r.Begin().Run(batch).End();                            // run.h:365-392, for the whole batch
//     r.Matches(i);  r.AcceptedRegexps(i);
//
// Pire::Gpu::Scanner also satisfies the reference's compile-time "Scanner concept"
// (pire/scanners/multi.h:137-194,:281-284) on the HOST in index space, so the
// reference's own templates -- Pire::Step, Pire::Run, Pire::Runner, LongestPrefix,
// ShortestPrefix (pire/run.h) -- compile against it unchanged; the parity tests use
// that to prove the ingest is lossless.  The host concept is for verification; the
// batch path never falls back to it.
//
// This header does not include any Pire header: the templated constructor only
// needs `sc.Save(std::ostream*)`.
#pragma once

#include <cstddef>
#include <cstdint>
#include <sstream>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "pire_b200.h"

namespace Pire {
namespace Gpu {

// Counterpart of Pire::Error (pire/stub/stl.h:213-217).
class Error : public std::runtime_error {
public:
    Error(int code, const std::string& what) : std::runtime_error(what), Code(code) {}
    int Code;
};

inline void Check(int rc, const char* where)
{
    if (rc != PIRE_GPU_OK)
        throw Error(rc, std::string(where) + ": " + pire_gpu_last_error());
}

// A batch of strings on the device: CSR offsets (n+1) or fixed length.
struct Batch {
    const uint8_t* Corpus;
    const uint64_t* Offsets;     // nullptr => fixed-length strings
    uint64_t FixedLen;
    uint64_t Count;
};

class Scanner {
public:
    // ---- Scanner concept (host, index space) --------------------------------
    typedef uint32_t State;
    typedef uint32_t Action;
    typedef unsigned short Char;     // Pire::Char, pire/defs.h:59

    Scanner() : Handle(nullptr), AcceptBegin(1, 0) {}

    // From a Scanner::Save() stream (multi.h:557-573).  device = -1: host only.
    Scanner(const void* image, size_t size, int device = 0) : Handle(nullptr)
    {
        Check(pire_gpu_scanner_create(image, size, device, &Handle), "pire_gpu_scanner_create");
        BuildAcceptCache();
    }

    // From any Pire scanner type whose Save() writes the multi-Scanner format
    // (Pire::Scanner, Pire::NonrelocScanner and their NoMask variants).
    template <class PireScanner>
    explicit Scanner(const PireScanner& sc, int device = 0) : Handle(nullptr)
    {
        std::ostringstream out;
        sc.Save(&out);
        const std::string image = out.str();
        Check(pire_gpu_scanner_create(image.data(), image.size(), device, &Handle), "pire_gpu_scanner_create");
        BuildAcceptCache();
    }

    Scanner(Scanner&& o) noexcept : Handle(o.Handle), AcceptBegin(std::move(o.AcceptBegin)), AcceptIds(std::move(o.AcceptIds))
    {
        o.Handle = nullptr;
        o.AcceptBegin.assign(1, 0);
    }
    Scanner& operator=(Scanner&& o) noexcept
    {
        if (this != &o) {
            pire_gpu_scanner_destroy(Handle);
            Handle = o.Handle;
            AcceptBegin = std::move(o.AcceptBegin);
            AcceptIds = std::move(o.AcceptIds);
            o.Handle = nullptr;
            o.AcceptBegin.assign(1, 0);
        }
        return *this;
    }
    Scanner(const Scanner&) = delete;
    Scanner& operator=(const Scanner&) = delete;
    ~Scanner() { pire_gpu_scanner_destroy(Handle); }

    size_t Size() const { return Info().states; }                       // multi.h:134
    bool Empty() const { return Info().empty != 0; }                    // multi.h:135
    size_t RegexpsCount() const { return Info().regexps; }              // multi.h:139
    size_t LettersCount() const { return Info().letters; }              // multi.h:140

    void Initialize(State& st) const { st = pire_gpu_initial(Handle); }                       // multi.h:161
    Action Next(State& st, Char c) const { st = pire_gpu_next(Handle, st, c); return 0; }     // multi.h:189-192
    void TakeAction(State&, Action) const {}                                                  // multi.h:194
    bool Final(const State& st) const { return pire_gpu_final(Handle, st) != 0; }             // multi.h:143
    bool Dead(const State& st) const { return pire_gpu_dead(Handle, st) != 0; }               // multi.h:147
    size_t StateIndex(State st) const { return st; }                                          // multi.h:281-284

    // multi.h:149-158.  The returned range stays valid for the scanner's lifetime.  The lists are built once in the
    // constructor, so this is a pure read: like a const Pire::Scanner, one object may be shared between threads.
    std::pair<const size_t*, const size_t*> AcceptedRegexps(const State& st) const
    {
        if (st >= AcceptBegin.size() - 1)
            return std::make_pair(AcceptIds.data(), AcceptIds.data());
        return std::make_pair(AcceptIds.data() + AcceptBegin[st], AcceptIds.data() + AcceptBegin[st + 1] - 1);
    }

    // ---- device ----------------------------------------------------------------
    void Tune(const Batch& sample, unsigned flags = PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END, void* stream = nullptr)
    {
        Check(pire_gpu_scanner_tune(Handle, sample.Corpus, sample.Offsets, sample.FixedLen, sample.Count, flags, stream),
              "pire_gpu_scanner_tune");
    }

    pire_gpu_info Info() const
    {
        pire_gpu_info info;
        Check(pire_gpu_scanner_info(Handle, &info), "pire_gpu_scanner_info");
        return info;
    }

    pire_gpu_scanner* Raw() const { return Handle; }

private:
    // every state's accept list, each followed by a terminator like m_final's (multi.h:96)
    void BuildAcceptCache()
    {
        const size_t states = Info().states;
        AcceptBegin.assign(states + 1, 0);
        AcceptIds.clear();
        std::vector<uint32_t> ids(64);
        for (size_t st = 0; st < states; ++st) {
            AcceptBegin[st] = AcceptIds.size();
            size_t k = pire_gpu_accepted_regexps(Handle, (uint32_t) st, ids.data(), ids.size());
            if (k > ids.size()) {
                ids.resize(k);
                k = pire_gpu_accepted_regexps(Handle, (uint32_t) st, ids.data(), ids.size());
            }
            AcceptIds.insert(AcceptIds.end(), ids.begin(), ids.begin() + k);
            AcceptIds.push_back(static_cast<size_t>(-1));
        }
        AcceptBegin[states] = AcceptIds.size();
    }

    pire_gpu_scanner* Handle;
    std::vector<size_t> AcceptBegin;      // [states + 1] into AcceptIds
    std::vector<size_t> AcceptIds;
};

// Counterpart of Pire::RunHelper (run.h:365-386) for a device batch.  Results are
// written to caller-owned device buffers (any may be null); MatchesHost() etc. are
// conveniences that copy them back through the host entry point.
// Runner(sc, st) for every string of the batch (pire_gpu_run_batch_from): the start states are n device words, tagged
// with From() so that a bare pointer is never taken for them, and the state output may be the same buffer, so that a
// batch of streams is carried on in place round after round:
//     Runner(gsc, BatchRunner::From(d_state)).Run(piece_k).Launch(nullptr, nullptr, d_state);          // round k
//     Runner(gsc, BatchRunner::From(d_state)).Run(last).End().Launch(d_bits, d_masks, d_state);        // the last one
class BatchRunner {
public:
    // n device words holding the StateIndex each string starts from (Runner(sc, st), run.h:391-392)
    struct StartWords {
        explicit StartWords(const uint32_t* d_words) : Words(d_words) {}
        const uint32_t* Words;
    };
    static StartWords From(const uint32_t* d_start) { return StartWords(d_start); }

    explicit BatchRunner(const Scanner& sc) : Sc(&sc), Start(nullptr), Flags(0), Ran(false) {}
    BatchRunner(const Scanner& sc, StartWords start) : BatchRunner(sc)
    {
        if (!start.Words)
            throw Error(PIRE_GPU_EINVAL, "BatchRunner::From needs device words");
        Start = start.Words;
    }

    BatchRunner& Begin() { Flags |= PIRE_GPU_RUN_BEGIN; return *this; }      // run.h:375
    BatchRunner& End() { Flags |= PIRE_GPU_RUN_END; return *this; }          // run.h:376
    BatchRunner& Run(const Batch& b) { Input = b; Ran = true; return *this; } // run.h:372

    // Launches the fused Begin/Run/End pass on `stream` (cudaStream_t as void*).
    void Launch(uint32_t* d_match_bits, uint32_t* d_accept_masks, uint32_t* d_state_idx, void* stream = nullptr) const
    {
        if (!Ran)
            throw Error(PIRE_GPU_EINVAL, "BatchRunner::Run() was not called");
        if (Start) {
            Check(pire_gpu_run_batch_from(Sc->Raw(), Input.Corpus, Input.Offsets, nullptr, Input.FixedLen, Input.Count, Flags, Start,
                                          d_match_bits, d_accept_masks, d_state_idx, stream),
                  "pire_gpu_run_batch_from");
            return;
        }
        Check(pire_gpu_run_batch(Sc->Raw(), Input.Corpus, Input.Offsets, Input.FixedLen, Input.Count, Flags, d_match_bits,
                                 d_accept_masks, d_state_idx, stream),
              "pire_gpu_run_batch");
    }

private:
    const Scanner* Sc;
    const uint32_t* Start;
    Batch Input;
    unsigned Flags;
    bool Ran;
};

inline BatchRunner Runner(const Scanner& sc) { return BatchRunner(sc); }     // run.h:388-389
// run.h:391-392, for every string of a batch
inline BatchRunner Runner(const Scanner& sc, BatchRunner::StartWords start) { return BatchRunner(sc, start); }

// Counterpart of Pire::RunHelper (run.h:365-392) for ONE string resident in HBM, scanned by the whole GPU
// (pire_gpu_run_string).  Run() may be called many times: the pieces are scanned as one string, the state carried in
// the caller-owned device word d_state (StateIndex, reference numbering), so chained calls do not synchronise.  Every
// call is asynchronous on `stream`; after End() the caller's device words hold the results (d_match_bits[0] bit 0 =
// Final(), d_accept_masks[0], *d_state), as pire_gpu_run_batch writes them for n = 1.
//     StringRunner r(gsc, d_state);                                // Runner(sc): from Initialize()
//     StringRunner r(gsc, StringRunner::From(d_start), d_state);   // Runner(sc, st): st in the device word d_start
//     r.Begin().Run(d_a, n_a).Run(d_b, n_b).End();
// The start word is tagged (From) so that it can never be taken for d_state or an output: every untagged call starts
// from Initialize().
class StringRunner {
public:
    // the device word holding the StateIndex a run starts from (Runner(sc, st), run.h:391-392)
    struct StartWord {
        explicit StartWord(const uint32_t* d_word) : Word(d_word) {}
        const uint32_t* Word;
    };
    static StartWord From(const uint32_t* d_start) { return StartWord(d_start); }

    StringRunner(const Scanner& sc, uint32_t* d_state, uint32_t* d_match_bits = nullptr, uint32_t* d_accept_masks = nullptr,
                 void* stream = nullptr)
        : Sc(&sc), Start(nullptr), State(d_state), Bits(d_match_bits), Masks(d_accept_masks), Stream(stream), Flags(0), Ran(false)
    {
        if (!d_state)
            throw Error(PIRE_GPU_EINVAL, "StringRunner needs a device word for its state");
    }
    // start.Word may be d_state: the state is then updated in place
    StringRunner(const Scanner& sc, StartWord start, uint32_t* d_state, uint32_t* d_match_bits = nullptr,
                 uint32_t* d_accept_masks = nullptr, void* stream = nullptr)
        : StringRunner(sc, d_state, d_match_bits, d_accept_masks, stream)
    {
        if (!start.Word)
            throw Error(PIRE_GPU_EINVAL, "StringRunner::From needs a device word");
        Start = start.Word;
    }

    StringRunner& Begin() { Flags |= PIRE_GPU_RUN_BEGIN; return *this; }                   // run.h:375, with the next launch
    StringRunner& Run(const uint8_t* d_text, uint64_t n) { Launch(d_text, n, 0); return *this; }   // run.h:372-373
    StringRunner& End() { Launch(nullptr, 0, PIRE_GPU_RUN_END); return *this; }             // run.h:376

private:
    void Launch(const uint8_t* d_text, uint64_t n, unsigned end)
    {
        Check(pire_gpu_run_string(Sc->Raw(), d_text, n, Flags | end, Ran ? State : Start, Bits, Masks, State, Stream),
              "pire_gpu_run_string");
        Flags = 0;
        Ran = true;
    }

    const Scanner* Sc;
    const uint32_t* Start;
    uint32_t* State;
    uint32_t* Bits;
    uint32_t* Masks;
    void* Stream;
    unsigned Flags;
    bool Ran;
};

// A Pire::HalfFinalScanner run over ONE string resident in HBM, counted by the whole GPU (pire_gpu_count_string):
// StringRunner's shape, with the counters of HalfFinalScanner::State.  Run() may be called many times: the pieces are
// counted as one string, the state carried in the caller-owned device word d_state and the counts ADDED to the
// caller-owned device array d_counts (max(1, RegexpsCount()) u64, zeroed by the caller before the first call), so
// chained calls do not synchronise.  After the stream is synchronised, d_counts[r] is State::Result(r)
// (half_final.h:88-90), *d_state the StateIndex reached and d_match_bits[0] bit 0 Final().  (This header needs no CUDA
// runtime, so reading the device words is the caller's.)
//     StringCounter c(gsc, d_counts, d_state);                                 // Initialize(), counted
//     StringCounter c(gsc, StringCounter::From(d_start), d_counts, d_state);   // resumed from st (not counted again)
//     c.Begin().Run(d_a, n_a).Run(d_b, n_b).End();
class StringCounter {
public:
    using StartWord = StringRunner::StartWord;
    static StartWord From(const uint32_t* d_start) { return StartWord(d_start); }

    StringCounter(const Scanner& sc, uint64_t* d_counts, uint32_t* d_state, uint32_t* d_match_bits = nullptr, void* stream = nullptr)
        : Sc(&sc), Start(nullptr), Counts(d_counts), State(d_state), Bits(d_match_bits), Stream(stream), Flags(0), Ran(false)
    {
        if (!d_counts || !d_state)
            throw Error(PIRE_GPU_EINVAL, "StringCounter needs device words for its counters and its state");
    }
    // start.Word may be d_state: the state is then updated in place
    StringCounter(const Scanner& sc, StartWord start, uint64_t* d_counts, uint32_t* d_state, uint32_t* d_match_bits = nullptr,
                  void* stream = nullptr)
        : StringCounter(sc, d_counts, d_state, d_match_bits, stream)
    {
        if (!start.Word)
            throw Error(PIRE_GPU_EINVAL, "StringCounter::From needs a device word");
        Start = start.Word;
    }

    StringCounter& Begin() { Flags |= PIRE_GPU_RUN_BEGIN; return *this; }
    StringCounter& Run(const uint8_t* d_text, uint64_t n) { Launch(d_text, n, 0); return *this; }
    StringCounter& End() { Launch(nullptr, 0, PIRE_GPU_RUN_END); return *this; }

private:
    void Launch(const uint8_t* d_text, uint64_t n, unsigned end)
    {
        Check(pire_gpu_count_string(Sc->Raw(), d_text, n, Flags | end, Ran ? State : Start, Counts, Bits, State, Stream),
              "pire_gpu_count_string");
        Flags = 0;
        Ran = true;
    }

    const Scanner* Sc;
    const uint32_t* Start;
    uint64_t* Counts;
    uint32_t* State;
    uint32_t* Bits;
    void* Stream;
    unsigned Flags;
    bool Ran;
};

// Where the matches StringCounter counts end (pire_gpu_match_ends_string): StringCounter's shape, with the entries
// (end, regexp id) appended in walk order to the caller-owned device arrays d_ends / d_ids (either may be null) of
// `capacity` entries, and their number ADDED to the caller-owned device word *d_found (zeroed by the caller before the
// first call).  Run() may be called many times: the pieces are one string, the state carried in d_state and the running
// byte offset kept here, so an end is the number of bytes of all pieces consumed when the state was entered, and chained
// calls do not synchronise.  End() is a launch of its own, at the total length.  After the stream is synchronised,
// *d_found is the number of entries (all of them, even past capacity) and the first min(*d_found, capacity) entries of
// d_ends / d_ids are the answer's first ones.
//     StringMatchEnds m(gsc, d_ends, d_ids, capacity, d_found, d_state);                                  // Initialize()
//     StringMatchEnds m(gsc, StringMatchEnds::From(d_start), d_ends, d_ids, capacity, d_found, d_state);  // resumed
//     m.Begin().Run(d_a, n_a).Run(d_b, n_b).End();
class StringMatchEnds;
class BatchMatchEnds;
void MatchStarts(const Scanner& rsc, const StringMatchEnds& ends, const uint8_t* d_window, uint64_t n_bytes, uint64_t base,
                 uint64_t* d_starts, uint8_t* d_open = nullptr, bool begin = true, bool end = true, uint64_t max_back = 0,
                 const uint64_t* d_first = nullptr);
void MatchStarts(const Scanner& rsc, const BatchMatchEnds& ends, const Batch& window, uint64_t* d_starts, uint8_t* d_open = nullptr,
                 bool begin = true, bool end = true, uint64_t max_back = 0, const uint64_t* d_first = nullptr);

class StringMatchEnds {
public:
    using StartWord = StringRunner::StartWord;
    static StartWord From(const uint32_t* d_start) { return StartWord(d_start); }

    StringMatchEnds(const Scanner& sc, uint64_t* d_ends, uint32_t* d_ids, uint64_t capacity, uint64_t* d_found, uint32_t* d_state,
                    uint32_t* d_match_bits = nullptr, void* stream = nullptr)
        : Sc(&sc), Start(nullptr), Ends(d_ends), Ids(d_ids), Capacity(capacity), Found(d_found), State(d_state), Bits(d_match_bits),
          Stream(stream), Base(0), Flags(0), Ran(false)
    {
        if (!d_found || !d_state)
            throw Error(PIRE_GPU_EINVAL, "StringMatchEnds needs device words for the number of entries and the state");
    }
    // start.Word may be d_state: the state is then updated in place
    StringMatchEnds(const Scanner& sc, StartWord start, uint64_t* d_ends, uint32_t* d_ids, uint64_t capacity, uint64_t* d_found,
                    uint32_t* d_state, uint32_t* d_match_bits = nullptr, void* stream = nullptr)
        : StringMatchEnds(sc, d_ends, d_ids, capacity, d_found, d_state, d_match_bits, stream)
    {
        if (!start.Word)
            throw Error(PIRE_GPU_EINVAL, "StringMatchEnds::From needs a device word");
        Start = start.Word;
    }

    StringMatchEnds& Begin() { Flags |= PIRE_GPU_RUN_BEGIN; return *this; }
    StringMatchEnds& Run(const uint8_t* d_text, uint64_t n) { Launch(d_text, n, 0); return *this; }
    StringMatchEnds& End() { Launch(nullptr, 0, PIRE_GPU_RUN_END); return *this; }

private:
    friend void MatchStarts(const Scanner&, const StringMatchEnds&, const uint8_t*, uint64_t, uint64_t, uint64_t*, uint8_t*, bool,
                            bool, uint64_t, const uint64_t*);
    void Launch(const uint8_t* d_text, uint64_t n, unsigned end)
    {
        Check(pire_gpu_match_ends_string(Sc->Raw(), d_text, n, Flags | end, Ran ? State : Start, Base, Ends, Ids, Capacity, Found,
                                         Bits, State, Stream),
              "pire_gpu_match_ends_string");
        Base += n;
        Flags = 0;
        Ran = true;
    }

    const Scanner* Sc;
    const uint32_t* Start;
    uint64_t* Ends;
    uint32_t* Ids;
    uint64_t Capacity;
    uint64_t* Found;
    uint32_t* State;
    uint32_t* Bits;
    void* Stream;
    uint64_t Base;
    unsigned Flags;
    bool Ran;
};

// StringCounter for n streams at once, one Pire::HalfFinalScanner::State each (pire_gpu_count_batch_from).  Every Run()
// launches at once on a batch of n strings, string i the next piece of stream i; the states are carried in the
// caller-owned device words d_state[0..n) and the counts ADDED to the caller-owned rows d_counts (n rows of
// max(1, RegexpsCount()) u64, zeroed by the caller before the first call), so chained calls do not synchronise.  After
// the stream is synchronised, d_counts[i * max(1, RegexpsCount()) + r] is stream i's State::Result(r), d_state[i] its
// StateIndex and bit i % 32 of d_match_bits[i / 32] its Final().  End() is a launch of its own over n empty strings.
//     BatchCounter c(gsc, n, d_counts, d_state);                                // Initialize(), counted
//     BatchCounter c(gsc, BatchCounter::From(d_start), n, d_counts, d_state);   // resumed from d_start[i] (not counted again)
//     c.Begin().Run(batch0).Run(batch1).End();
class BatchCounter {
public:
    using StartWords = BatchRunner::StartWords;
    static StartWords From(const uint32_t* d_start) { return StartWords(d_start); }

    BatchCounter(const Scanner& sc, uint64_t n, uint64_t* d_counts, uint32_t* d_state, uint32_t* d_match_bits = nullptr,
                 void* stream = nullptr)
        : Sc(&sc), N(n), Start(nullptr), Counts(d_counts), State(d_state), Bits(d_match_bits), Stream(stream), Flags(0), Ran(false)
    {
        if (n != 0 && (!d_counts || !d_state))
            throw Error(PIRE_GPU_EINVAL, "BatchCounter needs device words for its counters and its states");
    }
    // start.Words may be d_state: the states are then updated in place
    BatchCounter(const Scanner& sc, StartWords start, uint64_t n, uint64_t* d_counts, uint32_t* d_state,
                 uint32_t* d_match_bits = nullptr, void* stream = nullptr)
        : BatchCounter(sc, n, d_counts, d_state, d_match_bits, stream)
    {
        if (n != 0 && !start.Words)
            throw Error(PIRE_GPU_EINVAL, "BatchCounter::From needs device words");
        Start = start.Words;
    }

    BatchCounter& Begin() { Flags |= PIRE_GPU_RUN_BEGIN; return *this; }
    BatchCounter& Run(const Batch& b)
    {
        if (b.Count != N)
            throw Error(PIRE_GPU_EINVAL, "BatchCounter::Run needs a batch of n strings");
        Launch(b, 0);
        return *this;
    }
    BatchCounter& End()
    {
        const Batch empty = {nullptr, nullptr, 0, N};
        Launch(empty, PIRE_GPU_RUN_END);
        return *this;
    }

private:
    void Launch(const Batch& b, unsigned end)
    {
        Check(pire_gpu_count_batch_from(Sc->Raw(), b.Corpus, b.Offsets, b.FixedLen, b.Count, Flags | end, Ran ? State : Start,
                                        Counts, Bits, State, Stream),
              "pire_gpu_count_batch_from");
        Flags = 0;
        Ran = true;
    }

    const Scanner* Sc;
    uint64_t N;
    const uint32_t* Start;
    uint64_t* Counts;
    uint32_t* State;
    uint32_t* Bits;
    void* Stream;
    unsigned Flags;
    bool Ran;
};

// Where the matches BatchCounter counts end (pire_gpu_match_ends_batch_from): BatchCounter's shape, with the entries
// (stream, end, regexp id) appended to the caller-owned device arrays d_strings / d_ends / d_ids (each may be null) of
// `capacity` entries, ordered by stream within one Run() and in walk order within a stream, and their number ADDED to the
// caller-owned device word *d_found.  The states are carried in d_state[0..n) and the bytes each stream has consumed in
// d_pos[0..n) (both caller-owned; the caller zeroes *d_found and d_pos before the first call), so an end is the number of
// bytes of that stream consumed when the state was entered, and chained calls do not synchronise.  End() is a launch of
// its own over n empty strings.  After the stream is synchronised, *d_found is the number of entries (all of them, even
// past capacity), the first min(*d_found, capacity) entries are the answer's first ones, and d_state / d_match_bits are
// as BatchCounter's.
//     BatchMatchEnds m(gsc, n, d_pos, d_strings, d_ends, d_ids, capacity, d_found, d_state);                    // Initialize()
//     BatchMatchEnds m(gsc, BatchMatchEnds::From(d_start), n, d_pos, d_strings, d_ends, d_ids, capacity, d_found, d_state);
//     m.Begin().Run(batch0).Run(batch1).End();
class BatchMatchEnds {
public:
    using StartWords = BatchRunner::StartWords;
    static StartWords From(const uint32_t* d_start) { return StartWords(d_start); }

    BatchMatchEnds(const Scanner& sc, uint64_t n, uint64_t* d_pos, uint32_t* d_strings, uint64_t* d_ends, uint32_t* d_ids,
                   uint64_t capacity, uint64_t* d_found, uint32_t* d_state, uint32_t* d_match_bits = nullptr, void* stream = nullptr)
        : Sc(&sc), N(n), Start(nullptr), Pos(d_pos), Strings(d_strings), Ends(d_ends), Ids(d_ids), Capacity(capacity), Found(d_found),
          State(d_state), Bits(d_match_bits), Stream(stream), Flags(0), Ran(false)
    {
        if (!d_found || (n != 0 && (!d_pos || !d_state)))
            throw Error(PIRE_GPU_EINVAL, "BatchMatchEnds needs device words for the number of entries, the positions and the states");
    }
    // start.Words may be d_state: the states are then updated in place
    BatchMatchEnds(const Scanner& sc, StartWords start, uint64_t n, uint64_t* d_pos, uint32_t* d_strings, uint64_t* d_ends,
                   uint32_t* d_ids, uint64_t capacity, uint64_t* d_found, uint32_t* d_state, uint32_t* d_match_bits = nullptr,
                   void* stream = nullptr)
        : BatchMatchEnds(sc, n, d_pos, d_strings, d_ends, d_ids, capacity, d_found, d_state, d_match_bits, stream)
    {
        if (n != 0 && !start.Words)
            throw Error(PIRE_GPU_EINVAL, "BatchMatchEnds::From needs device words");
        Start = start.Words;
    }

    BatchMatchEnds& Begin() { Flags |= PIRE_GPU_RUN_BEGIN; return *this; }
    BatchMatchEnds& Run(const Batch& b)
    {
        if (b.Count != N)
            throw Error(PIRE_GPU_EINVAL, "BatchMatchEnds::Run needs a batch of n strings");
        Launch(b, 0);
        return *this;
    }
    BatchMatchEnds& End()
    {
        const Batch empty = {nullptr, nullptr, 0, N};
        Launch(empty, PIRE_GPU_RUN_END);
        return *this;
    }

private:
    friend void MatchStarts(const Scanner&, const BatchMatchEnds&, const Batch&, uint64_t*, uint8_t*, bool, bool, uint64_t,
                            const uint64_t*);
    void Launch(const Batch& b, unsigned end)
    {
        Check(pire_gpu_match_ends_batch_from(Sc->Raw(), b.Corpus, b.Offsets, b.FixedLen, b.Count, Flags | end, Ran ? State : Start,
                                             Pos, Strings, Ends, Ids, Capacity, Found, Bits, State, Stream),
              "pire_gpu_match_ends_batch_from");
        Flags = 0;
        Ran = true;
    }

    const Scanner* Sc;
    uint64_t N;
    const uint32_t* Start;
    uint64_t* Pos;
    uint32_t* Strings;
    uint64_t* Ends;
    uint32_t* Ids;
    uint64_t Capacity;
    uint64_t* Found;
    uint32_t* State;
    uint32_t* Bits;
    void* Stream;
    unsigned Flags;
    bool Ran;
};

// Where the matches of a StringMatchEnds / BatchMatchEnds start (pire_gpu_match_starts_string / _batch): Pire::LongestSuffix
// through `rsc`, the same patterns built with Fsm::Reverse() and glued in the same order, walked leftwards from each
// entry's end.  d_starts (and d_open, if given) get one word per entry of the ends' buffers, for entries
// [*d_first, min(*d_found, capacity)); entries whose end lies outside the window are not written.  String form: the
// window holds the text bytes at positions [base, base + n_bytes).  Batch form: the window is the batch of the ends'
// last round (string i ends where the ends' d_pos says).  begin: the window starts where the text begins; end: the
// ends' run took End().  On the ends' stream, with no synchronise.
//     StringMatchEnds m(gsc, d_ends, d_ids, cap, d_found, d_state);
//     m.Begin().Run(d_text, n).End();
//     MatchStarts(rsc, m, d_text, n, 0, d_starts);
inline void MatchStarts(const Scanner& rsc, const StringMatchEnds& ends, const uint8_t* d_window, uint64_t n_bytes, uint64_t base,
                        uint64_t* d_starts, uint8_t* d_open, bool begin, bool end, uint64_t max_back, const uint64_t* d_first)
{
    Check(pire_gpu_match_starts_string(rsc.Raw(), d_window, n_bytes, base, (begin ? PIRE_GPU_RUN_BEGIN : 0u) | (end ? PIRE_GPU_RUN_END : 0u),
                                       max_back, ends.Ends, ends.Ids, d_first, ends.Found, ends.Capacity, d_starts, d_open, ends.Stream),
          "pire_gpu_match_starts_string");
}

inline void MatchStarts(const Scanner& rsc, const BatchMatchEnds& ends, const Batch& window, uint64_t* d_starts, uint8_t* d_open,
                        bool begin, bool end, uint64_t max_back, const uint64_t* d_first)
{
    Check(pire_gpu_match_starts_batch(rsc.Raw(), window.Corpus, window.Offsets, window.FixedLen, window.Count, ends.Pos,
                                      (begin ? PIRE_GPU_RUN_BEGIN : 0u) | (end ? PIRE_GPU_RUN_END : 0u), max_back, ends.Strings,
                                      ends.Ends, ends.Ids, d_first, ends.Found, ends.Capacity, d_starts, d_open, ends.Stream),
          "pire_gpu_match_starts_batch");
}

// AcceptedRegexps for scanners with more than 32 regexps: rows of AcceptWords(sc) words, bit r of row i set iff
// regexp r is accepted by the state string i stopped in (d_state_idx from BatchRunner::Launch).
inline uint32_t AcceptWords(const Scanner& sc) { return pire_gpu_accept_words(sc.Raw()); }
inline void AcceptSets(const Scanner& sc, const uint32_t* d_state_idx, uint64_t n, uint32_t* d_sets, void* stream = nullptr)
{
    Check(pire_gpu_accept_sets(sc.Raw(), d_state_idx, n, d_sets, stream), "pire_gpu_accept_sets");
}

// One rank of a multi-GPU run (one GPU per process or thread): the communicator of pire_gpu_run_sharded.
//     rank 0:  unsigned char id[PIRE_GPU_COMM_ID_BYTES]; Comm::MakeId(id);  ... ship id to every rank ...
//     all:     Comm comm(id, world, rank, device);
//              comm.RunSharded(gsc, shard, n_global, flags, d_bits_all, d_masks, nullptr, stream);
class Comm {
public:
    static void MakeId(void* id) { Check(pire_gpu_comm_get_id(id), "pire_gpu_comm_get_id"); }
    Comm(const void* id, int world, int rank, int device) : Handle(nullptr)
    {
        Check(pire_gpu_comm_create(id, world, rank, device, &Handle), "pire_gpu_comm_create");
    }
    // around an ncclComm_t the caller owns (not destroyed here)
    Comm(void* ncclComm, int device) : Handle(nullptr) { Check(pire_gpu_comm_adopt(ncclComm, device, &Handle), "pire_gpu_comm_adopt"); }
    Comm(const Comm&) = delete;
    Comm& operator=(const Comm&) = delete;
    ~Comm() { pire_gpu_comm_destroy(Handle); }

    int World() const { int w = 1; pire_gpu_comm_info(Handle, &w, nullptr); return w; }
    int Rank() const { int r = 0; pire_gpu_comm_info(Handle, nullptr, &r); return r; }
    // [lo, hi) of this rank's shard and the words of the gathered bitmap
    std::pair<uint64_t, uint64_t> Bounds(uint64_t n_global) const
    {
        uint64_t lo = 0, hi = 0;
        pire_gpu_shard_bounds(n_global, World(), Rank(), &lo, &hi);
        return std::make_pair(lo, hi);
    }
    uint64_t Words(uint64_t n_global) const { return pire_gpu_sharded_words(n_global, World()); }

    // `shard` describes this rank's strings only (Count is ignored: the shard is Bounds(n_global)).
    void RunSharded(const Scanner& sc, const Batch& shard, uint64_t n_global, unsigned flags, uint32_t* d_match_bits_all,
                    uint32_t* d_accept_masks = nullptr, uint32_t* d_state_idx = nullptr, void* stream = nullptr)
    {
        Check(pire_gpu_run_sharded(sc.Raw(), Handle, shard.Corpus, shard.Offsets, shard.FixedLen, n_global, flags, d_match_bits_all,
                                   d_accept_masks, d_state_idx, stream), "pire_gpu_run_sharded");
    }
    void Wait(void* stream = nullptr) { Check(pire_gpu_comm_wait(Handle, stream), "pire_gpu_comm_wait"); }
    pire_gpu_comm* Raw() const { return Handle; }

private:
    pire_gpu_comm* Handle;
};

// Batch counterparts of Pire::LongestPrefix / Pire::ShortestPrefix (run.h:277-311): one prefix
// length per string into d_prefix_len (PIRE_GPU_NO_PREFIX where the reference returns null).
inline void LongestPrefix(const Scanner& sc, const Batch& b, uint32_t* d_prefix_len, bool throughBeginMark = false,
                          bool throughEndMark = false, void* stream = nullptr)
{
    unsigned flags = (throughBeginMark ? PIRE_GPU_RUN_BEGIN : 0u) | (throughEndMark ? PIRE_GPU_RUN_END : 0u);
    Check(pire_gpu_prefix_batch(sc.Raw(), b.Corpus, b.Offsets, b.FixedLen, b.Count, flags, 0, d_prefix_len, stream),
          "pire_gpu_prefix_batch");
}

inline void ShortestPrefix(const Scanner& sc, const Batch& b, uint32_t* d_prefix_len, bool throughBeginMark = false,
                           bool throughEndMark = false, void* stream = nullptr)
{
    unsigned flags = (throughBeginMark ? PIRE_GPU_RUN_BEGIN : 0u) | (throughEndMark ? PIRE_GPU_RUN_END : 0u);
    Check(pire_gpu_prefix_batch(sc.Raw(), b.Corpus, b.Offsets, b.FixedLen, b.Count, flags, 1, d_prefix_len, stream),
          "pire_gpu_prefix_batch");
}

// Batch counterparts of Pire::LongestSuffix / Pire::ShortestSuffix (run.h:316-362): every string is walked from
// its last byte to its first; one suffix length per string (PIRE_GPU_NO_PREFIX for null).
inline void LongestSuffix(const Scanner& sc, const Batch& b, uint32_t* d_suffix_len, bool throughEndMark = false,
                          bool throughBeginMark = false, void* stream = nullptr)
{
    unsigned flags = (throughBeginMark ? PIRE_GPU_RUN_BEGIN : 0u) | (throughEndMark ? PIRE_GPU_RUN_END : 0u);
    Check(pire_gpu_suffix_batch(sc.Raw(), b.Corpus, b.Offsets, b.FixedLen, b.Count, flags, 0, d_suffix_len, stream),
          "pire_gpu_suffix_batch");
}

inline void ShortestSuffix(const Scanner& sc, const Batch& b, uint32_t* d_suffix_len, bool throughEndMark = false,
                           bool throughBeginMark = false, void* stream = nullptr)
{
    unsigned flags = (throughBeginMark ? PIRE_GPU_RUN_BEGIN : 0u) | (throughEndMark ? PIRE_GPU_RUN_END : 0u);
    Check(pire_gpu_suffix_batch(sc.Raw(), b.Corpus, b.Offsets, b.FixedLen, b.Count, flags, 1, d_suffix_len, stream),
          "pire_gpu_suffix_batch");
}

// Batch counterpart of running a Pire::HalfFinalScanner over each string the way tests/count_ut.cpp:54-63
// does -- Initialize, [Step(BeginMark)], Run, [Step(EndMark)] -- and reading State::Result(r)
// (pire/scanners/half_final.h:88-90,:136-163) for every regexp: d_counts holds Count rows of
// max(1, RegexpsCount()) u32.  `sc` is built from the HalfFinalScanner (its Save() stream is Scanner's).
inline void HalfFinalCount(const Scanner& sc, const Batch& b, uint32_t* d_counts, uint32_t* d_match_bits = nullptr,
                           unsigned flags = PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END, void* stream = nullptr)
{
    Check(pire_gpu_count_batch(sc.Raw(), b.Corpus, b.Offsets, b.FixedLen, b.Count, flags, d_counts, d_match_bits, stream),
          "pire_gpu_count_batch");
}

// Host-buffer counterpart of `bool Pire::Runner(sc).Begin().Run(p, n).End()` for many
// strings at once (CSR): fills `matched[i]`.  With PIRE_GPU_RUN_LINES the offsets are those of a text's lines
// (std::getline), and the corpus is read up to offsets[n] - 1: a last line without '\n' ends at the text's end.
inline void MatchesHost(const Scanner& sc, const uint8_t* corpus, const uint64_t* offsets, uint64_t n,
                        std::vector<bool>& matched, unsigned flags = PIRE_GPU_RUN_BEGIN | PIRE_GPU_RUN_END)
{
    std::vector<uint32_t> bits((n + 31) / 32);
    const uint64_t bytes = n ? offsets[n] - ((flags & PIRE_GPU_RUN_LINES) ? 1 : 0) : 0;
    Check(pire_gpu_run_batch_host(sc.Raw(), corpus, bytes, offsets, 0, n, flags, bits.data(), nullptr, nullptr),
          "pire_gpu_run_batch_host");
    matched.resize(n);
    for (uint64_t i = 0; i < n; ++i)
        matched[i] = (bits[i / 32] >> (i % 32)) & 1u;
}

} // namespace Gpu
} // namespace Pire
