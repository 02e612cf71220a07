// oracle/ref_capi.cpp -- TEST INFRASTRUCTURE, not product code.
//
// A thin extern "C" face over the UNMODIFIED reference library (compiled from
// /root/reference by oracle/build_ref.sh into oracle/_ref/libpire_ref.so) so
// that Python tests and bench.py's CPU arm can:
//   * compile patterns exactly like tests/common.h:40-69 (ParseRegexp) and
//     tools/bench/bench.cpp:95-132 (CompileRe, incl. Scanner::Glue);
//   * serialise a compiled scanner with the reference's own Scanner::Save
//     (pire/scanners/multi.h:557-573) -- the byte stream the product ingests;
//   * run the reference's own hot path  Runner(sc).Begin().Run(p,n).End()
//     (pire/run.h:365-392) over a batch of strings, optionally on several
//     threads (the reference is single-threaded; a built scanner is immutable,
//     SURVEY.md 8(b) "Threading"), and report Final / AcceptedRegexps /
//     StateIndex per string.
// Nothing here is linked into, or called from, the product library.

#include <cstdint>
#include <cstring>
#include <sstream>
#include <string>
#include <thread>
#include <vector>
#include <stdexcept>

#include <pire.h>
#include <stub/stl.h>
#include <stub/memstreams.h>

namespace {

struct RefScanner {
	Pire::Scanner reloc;                      // Relocatable + ExitMasks<2> (what Save() writes)
	Pire::NonrelocScanner nonreloc;           // reference's fastest variant (multi.h:1119-1123)
	Pire::NonrelocScannerNoMask nonrelocNoMask;
	bool haveVariants = false;

	void MakeVariants()
	{
		if (haveVariants)
			return;
		nonreloc = Pire::NonrelocScanner(reloc);
		// NoMask variants differ in Shortcutting policy, so they cannot be
		// copy-converted (DeepCopy requires equal Shortcutting); they are
		// built by the compile/glue entry points below.
		haveVariants = true;
	}
};

void SetErr(char* err, size_t errlen, const char* what)
{
	if (err && errlen) {
		std::strncpy(err, what, errlen - 1);
		err[errlen - 1] = 0;
	}
}

// Same option letters as tests/common.h:40-58.
Pire::Fsm Parse(const char* pattern, const char* options)
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
	lexer.Encoding().FromLocal(pattern, pattern + std::strlen(pattern), std::back_inserter(ucs4));
	lexer.Assign(ucs4.begin(), ucs4.end());
	Pire::Fsm fsm = lexer.Parse();
	if (surround)
		fsm.Surround();
	if (reverse)
		fsm = fsm.Reverse();                         // tests/pire_ut.cpp:284: the scanner for suffix scans
	return fsm;
}

template<class Sc>
void RunRange(const Sc& sc, const uint8_t* corpus, const uint64_t* offsets, uint64_t fixedLen,
              uint64_t lo, uint64_t hi, int withBegin, int withEnd,
              uint8_t* finalOut, uint32_t* maskOut, uint32_t* stateOut)
{
	for (uint64_t i = lo; i < hi; ++i) {
		const char* b;
		const char* e;
		if (offsets) {
			b = (const char*) corpus + offsets[i];
			e = (const char*) corpus + offsets[i + 1];
		} else {
			b = (const char*) corpus + i * fixedLen;
			e = b + fixedLen;
		}
		Pire::RunHelper<Sc> r = Pire::Runner(sc);
		if (withBegin)
			r.Begin();
		r.Run(b, e);
		if (withEnd)
			r.End();
		typename Sc::State st = r.State();
		if (finalOut)
			finalOut[i] = sc.Final(st) ? 1 : 0;
		if (maskOut) {
			uint32_t m = 0;
			auto acc = sc.AcceptedRegexps(st);
			for (const size_t* p = acc.first; p != acc.second; ++p)
				if (*p < 32)
					m |= (1u << *p);
			maskOut[i] = m;
		}
		if (stateOut)
			stateOut[i] = (uint32_t) sc.StateIndex(st);
	}
}

template<class Sc>
void RunBatch(const Sc& sc, const uint8_t* corpus, const uint64_t* offsets, uint64_t fixedLen,
              uint64_t n, int withBegin, int withEnd, int threads,
              uint8_t* finalOut, uint32_t* maskOut, uint32_t* stateOut)
{
	if (threads <= 1 || n < 2) {
		RunRange(sc, corpus, offsets, fixedLen, 0, n, withBegin, withEnd, finalOut, maskOut, stateOut);
		return;
	}
	std::vector<std::thread> pool;
	uint64_t per = (n + threads - 1) / threads;
	for (int t = 0; t < threads; ++t) {
		uint64_t lo = std::min<uint64_t>(n, per * t), hi = std::min<uint64_t>(n, lo + per);
		if (lo == hi)
			break;
		pool.emplace_back([=, &sc] {
			RunRange(sc, corpus, offsets, fixedLen, lo, hi, withBegin, withEnd, finalOut, maskOut, stateOut);
		});
	}
	for (auto& th : pool)
		th.join();
}

// Index -> State needs the protected IndexToState (multi.h:447-450); a
// member-less subclass view gives access without touching the reference.
struct PeekScanner : Pire::Scanner {
	size_t ToState(size_t idx) const { return IndexToState(idx); }
};
const PeekScanner& AsPeek(const Pire::Scanner& sc) { return static_cast<const PeekScanner&>(sc); }

// ---- HalfFinalScanner (pire/scanners/half_final.h), the "next" row SURVEY.md 8(f) rank 3 ----
struct RefHalfFinal {
	Pire::HalfFinalScanner sc;
};

// The run of tests/count_ut.cpp:54-63: Initialize, [BeginMark], bytes, [EndMark]; then Result(i) per regexp.
void CountRange(const Pire::HalfFinalScanner& sc, const uint8_t* corpus, const uint64_t* offsets, uint64_t fixedLen,
                uint64_t lo, uint64_t hi, int withBegin, int withEnd, uint32_t* counts, uint8_t* finalOut)
{
	const size_t regs = sc.RegexpsCount();
	for (uint64_t i = lo; i < hi; ++i) {
		const char* b = offsets ? (const char*) corpus + offsets[i] : (const char*) corpus + i * fixedLen;
		const char* e = offsets ? (const char*) corpus + offsets[i + 1] : b + fixedLen;
		Pire::HalfFinalScanner::State st;
		sc.Initialize(st);
		if (withBegin)
			Pire::Step(sc, st, Pire::BeginMark);
		Pire::Run(sc, st, b, e);
		if (withEnd)
			Pire::Step(sc, st, Pire::EndMark);
		if (counts)
			for (size_t r = 0; r < regs; ++r)
				counts[i * regs + r] = (uint32_t) st.Result(r);
		if (finalOut)
			finalOut[i] = sc.Final(st) ? 1 : 0;
	}
}

} // namespace

extern "C" {

void* pref_compile(const char* pattern, const char* options, char* err, size_t errlen)
{
	try {
		Pire::Fsm fsm = Parse(pattern, options);
		RefScanner* h = new RefScanner;
		h->reloc = Pire::Fsm(fsm).Compile<Pire::Scanner>();
		h->nonrelocNoMask = Pire::Fsm(fsm).Compile<Pire::NonrelocScannerNoMask>();
		h->MakeVariants();
		return h;
	} catch (std::exception& e) {
		SetErr(err, errlen, e.what());
		return nullptr;
	}
}

// Scanner::Glue (multi.h:1092-1103).  On overflow the reference returns an
// Empty() scanner; we hand that back as a handle whose pref_empty() is 1.
void* pref_glue(void* a, void* b, size_t maxSize, char* err, size_t errlen)
{
	try {
		RefScanner* x = (RefScanner*) a;
		RefScanner* y = (RefScanner*) b;
		RefScanner* h = new RefScanner;
		h->reloc = Pire::Scanner::Glue(x->reloc, y->reloc, maxSize);
		h->nonrelocNoMask = Pire::NonrelocScannerNoMask::Glue(x->nonrelocNoMask, y->nonrelocNoMask, maxSize);
		h->MakeVariants();
		return h;
	} catch (std::exception& e) {
		SetErr(err, errlen, e.what());
		return nullptr;
	}
}

// A default-constructed (empty) scanner, multi.h:121.
void* pref_empty_scanner()
{
	RefScanner* h = new RefScanner;
	h->MakeVariants();
	return h;
}

void pref_free(void* h) { delete (RefScanner*) h; }

int pref_empty(void* h) { return ((RefScanner*) h)->reloc.Empty() ? 1 : 0; }
uint64_t pref_size(void* h) { return ((RefScanner*) h)->reloc.Size(); }
uint64_t pref_letters_count(void* h) { return ((RefScanner*) h)->reloc.LettersCount(); }
uint64_t pref_regexps_count(void* h) { return ((RefScanner*) h)->reloc.RegexpsCount(); }

uint64_t pref_initial_index(void* h)
{
	RefScanner* s = (RefScanner*) h;
	Pire::Scanner::State st;
	s->reloc.Initialize(st);
	return s->reloc.StateIndex(st);
}

// One Step() (run.h:50-57) in StateIndex space; ch may be BeginMark/EndMark.
uint64_t pref_next_index(void* h, uint64_t stateIndex, uint32_t ch)
{
	const PeekScanner& p = AsPeek(((RefScanner*) h)->reloc);
	Pire::Scanner::State cur = p.ToState(stateIndex);
	Pire::Step(p, cur, (Pire::Char) ch);
	return p.StateIndex(cur);
}

// Scanner::Save (multi.h:557-573).  Returns the stream length; copies it to buf
// when cap is large enough.
uint64_t pref_save(void* h, void* buf, uint64_t cap)
{
	std::ostringstream out;
	((RefScanner*) h)->reloc.Save(&out);
	std::string s = out.str();
	if (buf && cap >= s.size())
		std::memcpy(buf, s.data(), s.size());
	return s.size();
}

// variant: 0 = Scanner (reloc, ExitMasks), 1 = NonrelocScanner (ExitMasks),
//          2 = NonrelocScannerNoMask (pure table walk)
// offsets == NULL => fixed-length strings of fixedLen bytes, stride fixedLen.
int pref_run_batch(void* h, int variant, const uint8_t* corpus, const uint64_t* offsets,
                   uint64_t fixedLen, uint64_t n, int withBegin, int withEnd, int threads,
                   uint8_t* finalOut, uint32_t* maskOut, uint32_t* stateOut)
{
	RefScanner* s = (RefScanner*) h;
	switch (variant) {
	case 0: RunBatch(s->reloc, corpus, offsets, fixedLen, n, withBegin, withEnd, threads, finalOut, maskOut, stateOut); return 0;
	case 1: RunBatch(s->nonreloc, corpus, offsets, fixedLen, n, withBegin, withEnd, threads, finalOut, maskOut, stateOut); return 0;
	case 2: RunBatch(s->nonrelocNoMask, corpus, offsets, fixedLen, n, withBegin, withEnd, threads, finalOut, maskOut, stateOut); return 0;
	default: return -1;
	}
}

// AcceptedRegexps (multi.h:149-158) for a state index; returns the count.
uint64_t pref_accepted(void* h, uint64_t stateIndex, uint64_t* ids, uint64_t cap)
{
	const PeekScanner& p = AsPeek(((RefScanner*) h)->reloc);
	auto acc = p.AcceptedRegexps(p.ToState(stateIndex));
	uint64_t k = 0;
	for (const size_t* q = acc.first; q != acc.second; ++q, ++k)
		if (ids && k < cap)
			ids[k] = *q;
	return k;
}

int pref_final(void* h, uint64_t stateIndex)
{
	const PeekScanner& p = AsPeek(((RefScanner*) h)->reloc);
	return p.Final(p.ToState(stateIndex)) ? 1 : 0;
}

int pref_dead(void* h, uint64_t stateIndex)
{
	const PeekScanner& p = AsPeek(((RefScanner*) h)->reloc);
	return p.Dead(p.ToState(stateIndex)) ? 1 : 0;
}

// Pire::LongestPrefix / ShortestPrefix (run.h:277-311) per string.
// variant: 0 = Scanner (ExitMasks), 2 = NonrelocScannerNoMask (byte-by-byte predicates).
// out[i] = prefix length or -1 (the reference returns a null pointer).
int pref_prefix_batch(void* h, int variant, int shortest, const uint8_t* corpus, const uint64_t* offsets,
                      uint64_t fixedLen, uint64_t n, int throughBegin, int throughEnd, int64_t* out)
{
	RefScanner* s = (RefScanner*) h;
	for (uint64_t i = 0; i < n; ++i) {
		const char* b = (const char*) corpus + (offsets ? offsets[i] : i * fixedLen);
		const char* e = offsets ? (const char*) corpus + offsets[i + 1] : b + fixedLen;
		const char* p;
		if (variant == 0)
			p = shortest ? Pire::ShortestPrefix(s->reloc, b, e, throughBegin != 0, throughEnd != 0)
			             : Pire::LongestPrefix(s->reloc, b, e, throughBegin != 0, throughEnd != 0);
		else
			p = shortest ? Pire::ShortestPrefix(s->nonrelocNoMask, b, e, throughBegin != 0, throughEnd != 0)
			             : Pire::LongestPrefix(s->nonrelocNoMask, b, e, throughBegin != 0, throughEnd != 0);
		out[i] = p ? (int64_t) (p - b) : -1;
	}
	return 0;
}

// Pire::LongestSuffix / ShortestSuffix (run.h:316-362) per string, called the way tests/pire_ut.cpp:326-340 does:
// rbegin = the last byte, rend = one before the first.  out[i] = suffix length (rbegin - returned pointer) or -1.
int pref_suffix_batch(void* h, int variant, int shortest, const uint8_t* corpus, const uint64_t* offsets,
                      uint64_t fixedLen, uint64_t n, int throughEnd, int throughBegin, int64_t* out)
{
	RefScanner* s = (RefScanner*) h;
	for (uint64_t i = 0; i < n; ++i) {
		const char* b = (const char*) corpus + (offsets ? offsets[i] : i * fixedLen);
		const char* e = offsets ? (const char*) corpus + offsets[i + 1] : b + fixedLen;
		const char* rbegin = e - 1;
		const char* rend = b - 1;
		const char* p;
		if (variant == 0)
			p = shortest ? Pire::ShortestSuffix(s->reloc, rbegin, rend, throughEnd != 0, throughBegin != 0)
			             : Pire::LongestSuffix(s->reloc, rbegin, rend, throughEnd != 0, throughBegin != 0);
		else
			p = shortest ? Pire::ShortestSuffix(s->nonrelocNoMask, rbegin, rend, throughEnd != 0, throughBegin != 0)
			             : Pire::LongestSuffix(s->nonrelocNoMask, rbegin, rend, throughEnd != 0, throughBegin != 0);
		out[i] = p ? (int64_t) (rbegin - p) : -1;
	}
	return 0;
}

// mode 0: HalfFinalScanner(fsm) (half_final.h:38-46, MakeScanner);  modes 1..5: the counters of
// tests/count_ut.cpp:503-520 in that order -- MakeGreedyCounter(true), MakeGreedyCounter(false),
// MakeNonGreedyCounter(true,true), MakeNonGreedyCounter(true,false), MakeNonGreedyCounter(false).
void* pref_hf_compile(const char* pattern, const char* options, int mode, char* err, size_t errlen)
{
	try {
		Pire::Fsm fsm = Parse(pattern, options);
		RefHalfFinal* h = new RefHalfFinal;
		if (mode == 0) {
			h->sc = Pire::HalfFinalScanner(fsm);
		} else {
			Pire::HalfFinalFsm hf(fsm);
			switch (mode) {
			case 1: hf.MakeGreedyCounter(true); break;
			case 2: hf.MakeGreedyCounter(false); break;
			case 3: hf.MakeNonGreedyCounter(true, true); break;
			case 4: hf.MakeNonGreedyCounter(true, false); break;
			case 5: hf.MakeNonGreedyCounter(false); break;
			default: delete h; throw std::invalid_argument("unknown half-final mode");
			}
			h->sc = Pire::HalfFinalScanner(hf);
		}
		return h;
	} catch (std::exception& e) {
		SetErr(err, errlen, e.what());
		return nullptr;
	}
}

void* pref_hf_glue(void* a, void* b, size_t maxSize, char* err, size_t errlen)
{
	try {
		RefHalfFinal* h = new RefHalfFinal;
		h->sc = Pire::HalfFinalScanner::Glue(((RefHalfFinal*) a)->sc, ((RefHalfFinal*) b)->sc, maxSize);
		return h;
	} catch (std::exception& e) {
		SetErr(err, errlen, e.what());
		return nullptr;
	}
}

// Scanner::Load (multi.h:575-599) of a stored HalfFinalScanner image (it inherits Save/Load from Scanner).
void* pref_hf_load(const void* image, size_t size, char* err, size_t errlen)
{
	try {
		std::istringstream in(std::string((const char*) image, size));
		RefHalfFinal* h = new RefHalfFinal;
		h->sc.Load(&in);
		return h;
	} catch (std::exception& e) {
		SetErr(err, errlen, e.what());
		return nullptr;
	}
}

// Scanner::Load (multi.h:575-599) of a stored Pire::Scanner image (Relocatable, ExitMasks<2>).  Only variants 0 and 1
// answer for the handle: the NoMask variant cannot be made from a loaded image and stays empty.
void* pref_load(const void* image, size_t size, char* err, size_t errlen)
{
	try {
		std::istringstream in(std::string((const char*) image, size));
		RefScanner* h = new RefScanner;
		h->reloc.Load(&in);
		h->MakeVariants();
		return h;
	} catch (std::exception& e) {
		SetErr(err, errlen, e.what());
		return nullptr;
	}
}

void pref_hf_free(void* h) { delete (RefHalfFinal*) h; }
int pref_hf_empty(void* h) { return ((RefHalfFinal*) h)->sc.Empty() ? 1 : 0; }
uint64_t pref_hf_size(void* h) { return ((RefHalfFinal*) h)->sc.Size(); }
uint64_t pref_hf_regexps_count(void* h) { return ((RefHalfFinal*) h)->sc.RegexpsCount(); }

uint64_t pref_hf_save(void* h, void* buf, uint64_t cap)
{
	std::ostringstream out;
	((RefHalfFinal*) h)->sc.Save(&out);
	std::string s = out.str();
	if (buf && cap >= s.size())
		std::memcpy(buf, s.data(), s.size());
	return s.size();
}

// counts: n x RegexpsCount() u32, row per string.
int pref_hf_count_batch(void* h, const uint8_t* corpus, const uint64_t* offsets, uint64_t fixedLen, uint64_t n,
                        int withBegin, int withEnd, int threads, uint32_t* counts, uint8_t* finalOut)
{
	const Pire::HalfFinalScanner& sc = ((RefHalfFinal*) h)->sc;
	if (threads <= 1 || n < 2) {
		CountRange(sc, corpus, offsets, fixedLen, 0, n, withBegin, withEnd, counts, finalOut);
		return 0;
	}
	std::vector<std::thread> pool;
	uint64_t per = (n + threads - 1) / threads;
	for (int t = 0; t < threads; ++t) {
		uint64_t lo = std::min<uint64_t>(n, per * t), hi = std::min<uint64_t>(n, lo + per);
		if (lo == hi)
			break;
		pool.emplace_back([=, &sc] { CountRange(sc, corpus, offsets, fixedLen, lo, hi, withBegin, withEnd, counts, finalOut); });
	}
	for (auto& th : pool)
		th.join();
	return 0;
}

unsigned pref_hardware_threads() { return std::thread::hardware_concurrency(); }

} // extern "C"
