/* oracle/pire_oracle.c -- TEST INFRASTRUCTURE, not product code.
 * See pire_oracle.h.  Every function cites the reference lines it restates
 * (paths relative to the reference tree). */
#include "pire_oracle.h"

#include <string.h>

/* ---- serialised image -------------------------------------------------- */

/* pire/scanners/common.h:44-63 */
typedef struct {
    uint32_t magic, version, ptr_size, max_word_size, type, hdr_size;
} io_header;

/* pire/scanners/multi.h:315-323 (x86-64 layout, 48 bytes) */
typedef struct {
    uint32_t states, letters, regexps, pad0;
    uint64_t initial;
    uint32_t final_table_size, pad1;
    uint64_t relocation, shortcutting;
} io_locals;

static size_t align_up(size_t v, size_t b) { return (v + b - 1) & ~(b - 1); }

int pire_oracle_load(const void* blob, size_t size, pire_oracle_scanner* out)
{
    const uint8_t* p = (const uint8_t*) blob;
    io_header h;
    io_locals m;
    size_t pos = 0, bufsize;

    memset(out, 0, sizeof(*out));
    if (((uintptr_t) blob & 7) != 0)            /* common.h:89-93 CheckAlign */
        return -1;
    if (size < sizeof(h) + sizeof(m) + 8)
        return -2;
    memcpy(&h, p, sizeof(h));
    pos = align_up(sizeof(h), 8);
    /* common.h:65-78 Header::Validate */
    if (h.magic != 0x45524950u || h.ptr_size != 8 || h.max_word_size != 16)
        return -3;
    if (h.version != 7 && h.version != 6)
        return -4;
    if (h.type != 1 /* ScannerIOTypes::Scanner */ || h.hdr_size != sizeof(m))
        return -5;
    memcpy(&m, p + pos, sizeof(m));
    pos += align_up(sizeof(m), 8);
    if (m.relocation != 1)                      /* multi.h:56 Relocatable::Signature */
        return -6;
    out->empty = p[pos] ? 1 : 0;                /* multi.h:567-568 */
    pos += 8;
    out->states = m.states;
    out->letters = m.letters;
    out->regexps = m.regexps;
    out->final_table_size = m.final_table_size;
    out->initial = m.initial;
    out->shortcutting = m.shortcutting;
    if (m.shortcutting == 0x1000)               /* multi.h:828 NoShortcuts */
        out->header_cells = 2;                  /* 8-byte CommonRowHeader / 4 */
    else if (m.shortcutting == 0x2002)          /* multi.h:700 ExitMasks<2> */
        out->header_cells = 18;                 /* (8 masks + flags) * 8 / 4, multi.h:706-767 */
    else
        return -7;
    /* multi.h:347 RowSize: rows are multiples of 16 bytes = 4 cells */
    out->row_cells = (uint32_t) align_up(out->letters + out->header_cells, 4);
    if (out->empty)
        return 0;                               /* no image follows, multi.h:569-570 */
    /* multi.h:297-305 BufSize, :381-388 Markup */
    bufsize = align_up((size_t) PIRE_ORACLE_MAX_CHAR * 2
                       + (size_t) m.final_table_size * 8
                       + (size_t) m.states * 8
                       + (size_t) out->row_cells * m.states * 4, 8);
    if (size < pos + bufsize)
        return -8;
    out->letter_of = (const uint16_t*) (p + pos);
    out->final_tab = (const uint64_t*) (out->letter_of + PIRE_ORACLE_MAX_CHAR);
    out->final_idx = out->final_tab + m.final_table_size;
    out->trans = (const uint32_t*) (out->final_idx + m.states);
    return 0;
}

/* ---- per-state accessors ------------------------------------------------- */

static const uint64_t* row_header(const pire_oracle_scanner* sc, uint64_t st)
{
    return (const uint64_t*) ((const uint8_t*) sc->trans + st);
}

static uint64_t row_flags(const pire_oracle_scanner* sc, uint64_t st)
{
    /* ExitMasks<2>: 8 mask words precede Common.Flags (multi.h:763-767);
     * NoShortcuts: Flags is the whole header (multi.h:831-833). */
    return row_header(sc, st)[sc->header_cells == 18 ? 8 : 0];
}

uint64_t pire_oracle_initial(const pire_oracle_scanner* sc) { return sc->empty ? 0 : sc->initial; }

int pire_oracle_final(const pire_oracle_scanner* sc, uint64_t st)
{
    if (sc->empty) return 0;                    /* Null() = MakeFalse, multi.h:339-344 */
    return (row_flags(sc, st) & 1) != 0;        /* FinalFlag, multi.h:90-94,:143 */
}

int pire_oracle_dead(const pire_oracle_scanner* sc, uint64_t st)
{
    if (sc->empty) return 1;
    return (row_flags(sc, st) & 2) != 0;        /* DeadFlag, multi.h:147 */
}

uint64_t pire_oracle_state_index(const pire_oracle_scanner* sc, uint64_t st)
{
    if (sc->empty) return 0;
    return st / ((uint64_t) sc->row_cells * 4); /* multi.h:281-284 */
}

size_t pire_oracle_accepted(const pire_oracle_scanner* sc, uint64_t st, uint64_t* ids, size_t cap)
{
    const uint64_t* b;
    size_t k = 0;
    if (sc->empty) return 0;
    b = sc->final_tab + sc->final_idx[pire_oracle_state_index(sc, st)];
    for (; b[k] != (uint64_t) -1; ++k)          /* End terminator, multi.h:96,:154-156 */
        if (ids && k < cap)
            ids[k] = b[k];
    return k;
}

/* ---- the walk --------------------------------------------------------------- */

uint64_t pire_oracle_step(const pire_oracle_scanner* sc, uint64_t st, unsigned ch)
{
    uint16_t letter;
    int32_t shift;
    if (sc->empty) return 0;                    /* single never-final state */
    letter = sc->letter_of[ch];                 /* Translate, multi.h:163-166 */
    shift = (int32_t) ((const uint32_t*) ((const uint8_t*) sc->trans + st))[letter];
    return st + (int64_t) shift;                /* Relocatable::Go, multi.h:65; NextTranslated :177 */
}

uint64_t pire_oracle_run(const pire_oracle_scanner* sc, uint64_t st,
                         const uint8_t* begin, const uint8_t* end)
{
    /* run.h:186-226 splits [begin,end) into head/body/tail by address
     * alignment; every byte is fed through Step in order, which is all the
     * result depends on. */
    for (; begin != end; ++begin)
        st = pire_oracle_step(sc, st, *begin);
    return st;
}

static int word_has_byte(const uint8_t* w, uint64_t mask)
{
    /* platform.h:116-163 CheckBytes/IsAnySet: does any of 16 bytes equal the
     * mask's (replicated) byte? */
    uint8_t c = (uint8_t) mask;
    int i;
    for (i = 0; i < 16; ++i)
        if (w[i] == c) return 1;
    return 0;
}

uint64_t pire_oracle_run_shortcut(const pire_oracle_scanner* sc, uint64_t st,
                                  const uint8_t* begin, const uint8_t* end)
{
    const uint8_t* head = begin;
    const uint8_t* tail;
    int i;
    if (sc->empty || sc->header_cells != 18)
        return pire_oracle_run(sc, st, begin, end);
    tail = begin + ((size_t) (end - begin) & ~(size_t) 15);
    if (head == end)
        return st;
    /* multi.h:955-958: nothing but the marks can leave a NoExit state */
    if (row_header(sc, st)[0] == 2)
        return st;
    {
        int no_shortcut = row_header(sc, st)[0] == 1;       /* multi.h:964 */
        for (;;) {
            while (no_shortcut && head != tail) {              /* multi.h:968-975 */
                for (i = 0; i < 16; ++i)
                    st = pire_oracle_step(sc, st, head[i]);
                head += 16;
                no_shortcut = row_header(sc, st)[0] == 1;
            }
            if (head == tail)
                break;
            if (row_header(sc, st)[0] == 2)                    /* multi.h:979-982 */
                return st;
            {   /* multi.h:985 + :644-662: skip words with no exit byte */
                uint64_t m0 = row_header(sc, st)[0], m1 = row_header(sc, st)[4];
                while (head != tail && !word_has_byte(head, m0) && !word_has_byte(head, m1))
                    head += 16;
            }
            no_shortcut = 1;                                   /* multi.h:988 */
        }
    }
    for (; head != end; ++head)                                /* multi.h:991-996 + run.h tail */
        st = pire_oracle_step(sc, st, *head);
    return st;
}

void pire_oracle_run_batch(const pire_oracle_scanner* sc, const uint8_t* corpus,
                           const uint64_t* offsets, uint64_t fixed_len, uint64_t n,
                           int with_begin, int with_end, int use_shortcuts,
                           uint8_t* final_out, uint32_t* mask_out, uint32_t* state_out)
{
    uint64_t i;
    for (i = 0; i < n; ++i) {
        const uint8_t* b = offsets ? corpus + offsets[i] : corpus + i * fixed_len;
        const uint8_t* e = offsets ? corpus + offsets[i + 1] : b + fixed_len;
        uint64_t st = pire_oracle_initial(sc);                  /* RunHelper ctor, run.h:369 */
        if (with_begin)
            st = pire_oracle_step(sc, st, PIRE_ORACLE_BEGIN_MARK);   /* run.h:375 */
        st = use_shortcuts ? pire_oracle_run_shortcut(sc, st, b, e)
                           : pire_oracle_run(sc, st, b, e);     /* run.h:372-373 */
        if (with_end)
            st = pire_oracle_step(sc, st, PIRE_ORACLE_END_MARK);     /* run.h:376 */
        if (final_out)
            final_out[i] = (uint8_t) pire_oracle_final(sc, st);    /* run.h:380-381 */
        if (mask_out) {
            /* the whole accept list, however long (a list may name an id many times) */
            const uint64_t* it = sc->empty ? 0 : sc->final_tab + sc->final_idx[pire_oracle_state_index(sc, st)];
            uint32_t m = 0;
            for (; it && *it != (uint64_t) -1; ++it)
                if (*it < 32) m |= 1u << *it;
            mask_out[i] = m;
        }
        if (state_out)
            state_out[i] = (uint32_t) pire_oracle_state_index(sc, st);
    }
}

void pire_oracle_prefix_batch(const pire_oracle_scanner* sc, const uint8_t* corpus,
                              const uint64_t* offsets, uint64_t fixed_len, uint64_t n,
                              int through_begin, int through_end, int shortest, int64_t* out)
{
    uint64_t i;
    for (i = 0; i < n; ++i) {
        const uint8_t* b = offsets ? corpus + offsets[i] : corpus + i * fixed_len;
        const uint8_t* e = offsets ? corpus + offsets[i + 1] : b + fixed_len;
        const uint8_t* p;
        uint64_t st = pire_oracle_initial(sc);                          /* run.h:280-281 / :297-298 */
        int64_t pos = -1;
        int stop = 0;
        if (through_begin)
            st = pire_oracle_step(sc, st, PIRE_ORACLE_BEGIN_MARK);      /* run.h:282-283 / :299-300 */
        if (pire_oracle_final(sc, st)) {                                /* run.h:284 / :301-302 */
            pos = 0;
            stop = shortest;
        }
        for (p = b; p != e && !stop; ++p) {
            st = pire_oracle_step(sc, st, *p);
            if (pire_oracle_final(sc, st)) {                            /* LongestPrefixPred run.h:92-93, Shortest :76-79 */
                pos = (int64_t) (p + 1 - b);
                if (shortest)
                    stop = 1;
            }
            if (!stop && pire_oracle_dead(sc, st))                      /* run.h:82 / :94 */
                stop = 1;
        }
        if (through_end) {                                              /* run.h:286-290 / :305-309 */
            st = pire_oracle_step(sc, st, PIRE_ORACLE_END_MARK);
            if (pire_oracle_final(sc, st) && (!shortest || pos < 0))
                pos = (int64_t) (e - b);
        }
        out[i] = pos;
    }
}

/* LongestSuffix / ShortestSuffix, run.h:316-362: the string is walked from its last byte to its first. */
void pire_oracle_suffix_batch(const pire_oracle_scanner* sc, const uint8_t* corpus,
                              const uint64_t* offsets, uint64_t fixed_len, uint64_t n,
                              int through_end, int through_begin, int shortest, int64_t* out)
{
    uint64_t i;
    for (i = 0; i < n; ++i) {
        const uint8_t* b = offsets ? corpus + offsets[i] : corpus + i * fixed_len;
        const uint8_t* e = offsets ? corpus + offsets[i + 1] : b + fixed_len;
        const uint8_t* rbegin = e;                 /* one past the next byte to read (the reference's rbegin + 1) */
        uint64_t st = pire_oracle_initial(sc);
        int64_t pos = -1;
        if (through_end)
            st = pire_oracle_step(sc, st, PIRE_ORACLE_END_MARK);            /* run.h:321-322 / :350-351 */
        if (shortest) {
            /* run.h:353-360 */
            while (rbegin != b && !pire_oracle_final(sc, st) && !pire_oracle_dead(sc, st)) {
                --rbegin;
                st = pire_oracle_step(sc, st, *rbegin);
            }
            if (through_begin)
                st = pire_oracle_step(sc, st, PIRE_ORACLE_BEGIN_MARK);      /* from wherever the scan stopped */
            if (pire_oracle_final(sc, st))
                pos = (int64_t) (e - rbegin);
        } else {
            /* run.h:327-340 */
            while (rbegin != b && !pire_oracle_dead(sc, st)) {
                if (pire_oracle_final(sc, st))
                    pos = (int64_t) (e - rbegin);
                --rbegin;
                st = pire_oracle_step(sc, st, *rbegin);
            }
            if (pire_oracle_final(sc, st))
                pos = (int64_t) (e - rbegin);
            if (through_begin) {
                st = pire_oracle_step(sc, st, PIRE_ORACLE_BEGIN_MARK);
                if (pire_oracle_final(sc, st))
                    pos = (int64_t) (e - rbegin);
            }
        }
        out[i] = pos;
    }
}

/* ---- HalfFinalScanner counting (pire/scanners/half_final.h) ------------------------------- */

/* TakeAction, half_final.h:154-163: in a final state every entry of the state's accept list bumps the
 * counter of the regexp it names (an id may be listed several times: BuildFinals, half_final.h:215-226). */
static void oracle_take_action(const pire_oracle_scanner* sc, uint64_t st, uint32_t* row)
{
    const uint64_t* it;
    if (sc->empty || !pire_oracle_final(sc, st))
        return;
    for (it = sc->final_tab + sc->final_idx[pire_oracle_state_index(sc, st)]; *it != (uint64_t) -1; ++it)
        if (*it < sc->regexps)
            row[*it]++;
}

void pire_oracle_count_batch(const pire_oracle_scanner* sc, const uint8_t* corpus,
                             const uint64_t* offsets, uint64_t fixed_len, uint64_t n,
                             int with_begin, int with_end, uint32_t* counts, uint8_t* final_out)
{
    uint64_t i;
    const uint32_t regs = sc->regexps ? sc->regexps : 1;
    for (i = 0; i < n; ++i) {
        const uint8_t* b = offsets ? corpus + offsets[i] : corpus + i * fixed_len;
        const uint8_t* e = offsets ? corpus + offsets[i + 1] : b + fixed_len;
        const uint8_t* p;
        uint32_t* row = counts + i * regs;
        uint64_t st = pire_oracle_initial(sc);             /* Initialize, half_final.h:136-141 ... */
        memset(row, 0, regs * sizeof(uint32_t));
        oracle_take_action(sc, st, row);                   /* ... which ends in TakeAction(state, 0) */
        if (with_begin) {                                  /* Step = Next + TakeAction, run.h:50-57 */
            st = pire_oracle_step(sc, st, PIRE_ORACLE_BEGIN_MARK);
            oracle_take_action(sc, st, row);
        }
        for (p = b; p != e; ++p) {
            st = pire_oracle_step(sc, st, *p);
            oracle_take_action(sc, st, row);
        }
        if (with_end) {
            st = pire_oracle_step(sc, st, PIRE_ORACLE_END_MARK);
            oracle_take_action(sc, st, row);
        }
        if (final_out)
            final_out[i] = (uint8_t) pire_oracle_final(sc, st);
    }
}
