"""Synthesized automata for differential tests (TEST INFRASTRUCTURE; nothing under pire_b200/ imports this module).

Every GPU test elsewhere runs on automata that came out of Pire's regex compiler, and compiled regexes make a narrow
family of tables.  The kernels branch on properties of the table instead -- the hot set and its final partition, the
look-ahead filter, 16- or 32-bit cells, packed counters, the ``live`` table -- so this module writes the automaton
itself, from a seed, and checks the GPU against a plain walker over the generator's own tables:

* ``Dfa``: ``states``, the 256 bytes partitioned into letter classes, one class for BeginMark and one for EndMark,
  ``next[state][class]``, finals, accept lists, ``initial`` and ``regexps``.
* ``Dfa.image()``: a version 7, Relocatable, ExitMasks<2> ``Scanner::Save()`` image of it.  The letter slots follow
  real images: slots 256 and 260-263 share one class that no byte has, slot 257 (Epsilon) holds 0, and each mark has
  a class of its own.  Row headers carry the exit masks (NoExit, one or two exit bytes, otherwise no shortcut) and the
  Final and Dead flags, Dead meaning unreachable from the initial state or with no final state reachable.
* the walker (``run``, ``count``, ``match_ends``, ``prefix``, ``suffix``, ``match_starts``): numpy, vectorised over the
  strings of a batch, over ``next`` and the class table -- never over the image bytes.
* the families: functions of a seed that each assert the property they promise (state counts at the hot-set and
  width edges, ``look_ok`` false, weight-15 accept lists, the convergence distance of shift registers).
"""
import struct
import numpy as np

BEGIN_MARK, END_MARK = 258, 259
MAX_CHAR = 264
HEADER_CELLS = 18                       # ExitMasks<2>: 2 masks x 4 size_t + Flags, in 4-byte cells
NO_SHORTCUT, NO_EXIT = 1, 2
MAX_HOT, PRIV_ROWS, PRIV_HOT_ROWS = 255, 48, 115
UNKNOWN = 0xFFFFFFFF


def _round_up(v, b):
    return (v + b - 1) // b * b


class Dfa:
    """A complete deterministic automaton over byte classes.  ``cls[b]`` is the class of byte b (0..L-1); class L is
    the byteless class of slots 256 and 260-263, L + 1 BeginMark's and L + 2 EndMark's, so ``letters = L + 3``.
    ``accept[s]`` is the accept list of state s (repeats allowed).  ``nxt[s, L]`` is s itself: nothing steps it."""

    def __init__(self, name, nxt, cls, final, accept, initial, regexps):
        self.name = name
        self.nxt = np.ascontiguousarray(nxt, dtype=np.int64)
        self.cls = np.ascontiguousarray(cls, dtype=np.int64)
        self.states, self.letters = self.nxt.shape
        self.L = self.letters - 3
        self.begin_cls, self.end_cls = self.L + 1, self.L + 2
        assert self.cls.shape == (256,) and self.cls.min() >= 0 and self.cls.max() < self.L
        assert (self.nxt[:, self.L] == np.arange(self.states)).all()
        self.final = np.ascontiguousarray(final, dtype=bool)
        self.accept = [list(map(int, a)) for a in accept]
        assert len(self.accept) == self.states
        self.initial, self.regexps = int(initial), int(regexps)
        self.dead = self._dead()
        self._live = None

    # ------------------------------------------------------------------------------------------- derived tables
    def step(self, s, ch):
        """One step on a byte (0..255) or a mark (258, 259)."""
        c = self.begin_cls if ch == BEGIN_MARK else self.end_cls if ch == END_MARK else self.cls[ch]
        return int(self.nxt[s, c])

    def _dead(self):
        """Fsm::DeadStates over all letters: not reachable from the initial state, or no final state reachable."""
        S = self.states
        src = np.repeat(np.arange(S), self.letters)
        dst = self.nxt.reshape(-1)
        fwd = _reach(S, src, dst, [self.initial])
        back = _reach(S, dst, src, np.nonzero(self.final)[0])
        return ~(fwd & back)

    def acc_csr(self, finals_only, limit):
        """Accept lists as CSR (begin[S + 1], ids): with ``finals_only`` the lists TakeAction reads; ids < limit."""
        begin = np.zeros(self.states + 1, np.int64)
        ids = []
        for s in range(self.states):
            if not finals_only or self.final[s]:
                ids.extend(i for i in self.accept[s] if i < limit)
            begin[s + 1] = len(ids)
        return begin, np.asarray(ids, np.int64)

    def masks32(self):
        """AcceptedRegexps as a bit mask of the ids below 32, per state (any state, final or not)."""
        m = np.zeros(self.states, np.uint32)
        for s, a in enumerate(self.accept):
            for i in a:
                if i < 32:
                    m[s] |= np.uint32(1 << i)
        return m

    def weights(self):
        """weights[s, r]: how many times a TakeAction in s adds to counter r (0 unless s is final)."""
        R = max(1, self.regexps)
        w = np.zeros((self.states, R), np.int64)
        for s in np.nonzero(self.final)[0]:
            for i in self.accept[s]:
                if i < R:
                    w[s, i] += 1
        return w

    def live(self):
        """live[s]: the set of ids some walk from s (over bytes and marks) still accepts, as a bool [S, R] array."""
        if self._live is None:
            R = max(1, self.regexps)
            live = self.weights() > 0
            pred = [[] for _ in range(self.states)]
            for s in range(self.states):
                for t in set(self.nxt[s].tolist()):
                    pred[t].append(s)
            work = list(range(self.states))
            while work:
                t = work.pop()
                for s in pred[t]:
                    grow = live[t] & ~live[s]
                    if grow.any():
                        live[s] |= grow
                        work.append(s)
            assert live.shape == (self.states, R)
            self._live = live
        return self._live

    def static_hot_order(self):
        """The order dfa_tables.cpp ranks rows in without a tuning sample: Begin()'s state, Initialize()'s, breadth
        first over the bytes, then every state no byte reaches in index order.  Returns (order, byte-reachable count)."""
        seen = np.zeros(self.states, bool)
        order = []
        for s in (self.step(self.initial, BEGIN_MARK), self.initial):
            if not seen[s]:
                seen[s] = True
                order.append(s)
        head = 0
        while head < len(order):
            for t in self.nxt[order[head], self.cls].tolist():           # children in byte order
                if not seen[t]:
                    seen[t] = True
                    order.append(t)
            head += 1
        reached = len(order)
        order.extend(np.nonzero(~seen)[0].tolist())
        return order, reached

    def hot_layout(self, max_hot=MAX_HOT):
        """The renumbering of BuildScanTables for the static order: (new_of_old, H, first_final_hot, look_ok)."""
        order, _ = self.static_hot_order()
        H = max(1, min(MAX_HOT, max_hot, self.states))
        hot = order[:H]
        hot = [s for s in hot if not self.final[s]] + [s for s in hot if self.final[s]]
        first_final = next((k for k, s in enumerate(hot) if self.final[s]), len(hot))
        new = np.full(self.states, -1, np.int64)
        new[hot] = np.arange(H)
        rest = np.nonzero(new < 0)[0]
        new[rest] = np.arange(H, self.states)
        look_ok = True
        g1 = new[self.nxt[hot[0], self.cls]]
        for b in range(256):
            if g1[b] != 0 and g1[b] >= H:
                look_ok = False
        return new, H, first_final, look_ok

    # ----------------------------------------------------------------------------------------------- the image
    def image(self):
        """A Scanner::Save() stream: version 7, Relocatable, ExitMasks<2>."""
        S, letters, L = self.states, self.letters, self.L
        row_cells = _round_up(letters + HEADER_CELLS, 4)
        row_bytes = row_cells * 4
        slots = np.zeros(MAX_CHAR, np.uint16)
        slots[:256] = HEADER_CELLS + self.cls
        slots[[256, 260, 261, 262, 263]] = HEADER_CELLS + L
        slots[257] = 0
        slots[BEGIN_MARK] = HEADER_CELLS + self.begin_cls
        slots[END_MARK] = HEADER_CELLS + self.end_cls
        final_idx = np.zeros(S, np.uint64)
        table = []
        for s in range(S):
            final_idx[s] = len(table)
            table.extend(self.accept[s])
            table.append(0xFFFFFFFFFFFFFFFF)
        table = np.asarray(table, np.uint64)
        rows = np.zeros((S, row_cells), np.uint32)
        rows[:, HEADER_CELLS:HEADER_CELLS + letters] = ((self.nxt - np.arange(S)[:, None]) * row_bytes).astype(np.int64).astype(
            np.uint32)
        header = rows[:, :HEADER_CELLS].view(np.uint64)          # [S, 9]: mask words 0-3, 4-7, flags 8
        header[:, 8] = self.final.astype(np.uint64) | (self.dead.astype(np.uint64) << np.uint64(1))
        m0, m1 = self._exit_masks()
        header[:, 0:4] = m0[:, None]
        header[:, 4:8] = m1[:, None]
        out = struct.pack("<6I", 0x45524950, 7, 8, 16, 1, 48)
        out += struct.pack("<IIIIQIIQQ", S, letters, self.regexps, 0, self.initial * row_bytes, len(table), 0, 1, 0x2002)
        out += struct.pack("<Q", 0)                              # Empty() == false, padded to 8 bytes
        body = slots.tobytes() + table.tobytes() + final_idx.tobytes() + rows.tobytes()
        return out + body + bytes(_round_up(len(body), 8) - len(body))

    def _exit_masks(self):
        """BuildShortcuts for ExitMasks<2>: each byte on which a row leaves itself takes a mask (its value in every
        byte of the word), classes in column order; more than two such bytes is no shortcut, none is NoExit."""
        S = self.states
        fill = np.uint64(0x0101010101010101)
        bytes_of = [np.nonzero(self.cls == c)[0] for c in range(self.letters)]
        leaves = self.nxt != np.arange(S)[:, None]
        m0 = np.full(S, NO_EXIT, np.uint64)
        m1 = np.zeros(S, np.uint64)
        for s in range(S):
            masks = [NO_EXIT, NO_SHORTCUT]
            ind, broke = 0, False
            for c in np.nonzero(leaves[s])[0]:
                chars = bytes_of[c]
                if ind + len(chars) > 2:
                    broke = True
                    break
                for ch in chars:
                    masks[ind] = int(ch) * int(fill)
                    ind += 1
            if broke:
                masks[0] = NO_SHORTCUT
            ind = max(ind, 1)
            for k in range(ind, 2):
                masks[k] = masks[ind - 1]
            m0[s], m1[s] = masks
        return m0, m1

    # -------------------------------------------------------------------------------------------------- the walker
    def paths(self, strings, starts=None, begin=True):
        """Walk every string: P[i, j] = the state after j bytes of string i (j <= len_i), from its start (Initialize()
        when ``starts`` is None, else starts[i]) after BeginMark when ``begin``.  Rows of unknown starts (>= states)
        are -1.  Returns (P, lengths, start states before BeginMark)."""
        n = len(strings)
        lens = np.array([len(s) for s in strings], np.int64)
        width = int(lens.max()) if n else 0
        mat = np.zeros((n, width), np.uint8)
        for i, s in enumerate(strings):
            mat[i, : len(s)] = np.frombuffer(s, np.uint8)
        s0 = np.full(n, self.initial, np.int64) if starts is None else np.asarray(starts, np.int64).copy()
        known = s0 < self.states
        P = np.full((n, width + 1), -1, np.int64)
        cur = np.where(known, s0, 0)
        if begin:
            cur = self.nxt[cur, self.begin_cls]
        P[:, 0] = np.where(known, cur, -1)
        if n == 1 and width > 4096:                             # one long string: a plain loop beats numpy steps
            nxt = self.nxt.tolist()
            cl = self.cls.tolist()
            st = int(cur[0])
            out = P[0]
            if known[0]:
                for j, b in enumerate(strings[0]):
                    st = nxt[st][cl[b]]
                    out[j + 1] = st
            return P, lens, np.where(known, s0, -1)
        cls = self.cls[mat]
        for j in range(width):
            go = known & (lens > j)
            cur = np.where(go, self.nxt[cur, cls[:, j]], cur)
            P[:, j + 1] = np.where(go, cur, -1)
        return P, lens, np.where(known, s0, -1)

    def run(self, strings, starts=None, begin=True, end=True):
        """Runner(sc[, st]) [.Begin()] .Run(s) [.End()]: (final u8, accept mask u32, StateIndex u32) per string."""
        P, lens, s0 = self.paths(strings, starts, begin)
        n = len(strings)
        last = P[np.arange(n), lens] if n else np.zeros(0, np.int64)
        known = s0 >= 0
        if end:
            last = np.where(known, self.nxt[np.maximum(last, 0), self.end_cls], -1)
        fin = np.where(known, self.final[np.maximum(last, 0)], False).astype(np.uint8)
        mask = np.where(known, self.masks32()[np.maximum(last, 0)], 0).astype(np.uint32)
        state = np.where(known, last, UNKNOWN).astype(np.uint32)
        return fin, mask, state

    def _events(self, strings, starts, begin, end):
        """Every TakeAction of the HalfFinalScanner run, in walk order: (string, position, state) arrays sorted by
        string and then step.  A fresh start (``starts`` None) takes Initialize()'s, a resumed one does not."""
        P, lens, s0 = self.paths(strings, starts, begin)
        n = len(strings)
        ev_s, ev_p, ev_k, ev_st = [], [], [], []
        known = s0 >= 0
        idx = np.arange(n)
        if starts is None:
            ev_s.append(idx); ev_p.append(np.zeros(n, np.int64)); ev_k.append(np.zeros(n, np.int64)); ev_st.append(s0)
        if begin:
            ev_s.append(idx[known]); ev_p.append(np.zeros(int(known.sum()), np.int64))
            ev_k.append(np.ones(int(known.sum()), np.int64)); ev_st.append(P[known, 0])
        valid = (np.arange(P.shape[1] - 1)[None, :] < lens[:, None]) & known[:, None]
        ii, jj = np.nonzero(valid)
        ev_s.append(ii); ev_p.append(jj + 1); ev_k.append(jj + 2); ev_st.append(P[ii, jj + 1])
        last = P[idx, lens] if n else np.zeros(0, np.int64)
        if end:
            e = np.where(known, self.nxt[np.maximum(last, 0), self.end_cls], -1)
            ev_s.append(idx[known]); ev_p.append(lens[known]); ev_k.append(lens[known] + 2); ev_st.append(e[known])
            last = e
        s, p, k, st = (np.concatenate(x) if x else np.zeros(0, np.int64) for x in (ev_s, ev_p, ev_k, ev_st))
        keep = st >= 0
        s, p, k, st = s[keep], p[keep], k[keep], st[keep]
        order = np.lexsort((k, s))
        fin = np.where(known, self.final[np.maximum(last, 0)], False).astype(np.uint8)
        state = np.where(known, last, UNKNOWN).astype(np.uint32)
        return s[order], p[order], st[order], fin, state

    def count(self, strings, starts=None, begin=True, end=True):
        """HalfFinalScanner counts: (counts[n, max(1, regexps)] int64, final u8, StateIndex u32)."""
        s, _, st, fin, state = self._events(strings, starts, begin, end)
        W = self.weights()
        counts = np.zeros((len(strings), W.shape[1]), np.int64)
        np.add.at(counts, s, W[st])
        return counts, fin, state

    def match_ends(self, strings, starts=None, begin=True, end=True, bases=None):
        """Every TakeAction's entries (string, end, id) in walk order, ids in accept-list order; end = base + the
        bytes consumed.  Returns (strings u32, ends u64, ids u32, final u8, StateIndex u32)."""
        s, p, st, fin, state = self._events(strings, starts, begin, end)
        ab, ai = self.acc_csr(True, max(1, self.regexps))
        cnt = ab[st + 1] - ab[st]
        rs = np.repeat(s, cnt)
        rp = np.repeat(p, cnt)
        first = np.repeat(ab[st], cnt)
        within = np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        ids = ai[first + within] if len(ai) else np.zeros(0, np.int64)
        if bases is not None:
            rp = rp + np.asarray(bases, np.int64)[rs]
        return rs.astype(np.uint32), rp.astype(np.uint64), ids.astype(np.uint32), fin, state

    def prefix(self, strings, shortest=False, through_begin=False, through_end=False):
        """LongestPrefix / ShortestPrefix with the byte-by-byte predicates and the Dead stop: length or -1."""
        P, lens, _ = self.paths(strings, None, through_begin)
        n, W = P.shape[0], P.shape[1] - 1
        out = np.full(n, -1, np.int64)
        for i in range(n):
            row = P[i, : lens[i] + 1]
            fin, dead = self.final[row], self.dead[row]
            pos, stop_at = -1, lens[i]
            if fin[0]:
                pos = 0
                if shortest:
                    stop_at = 0
            if not (shortest and fin[0]):
                for j in range(1, lens[i] + 1):
                    if fin[j]:
                        pos = j
                        if shortest:
                            stop_at = j
                            break
                    if dead[j]:
                        stop_at = j
                        break
            if through_end:
                e = self.nxt[row[stop_at], self.end_cls]
                if self.final[e] and (not shortest or pos < 0):
                    pos = int(lens[i])
            out[i] = pos
        return out

    def suffix(self, strings, shortest=False, through_end=False, through_begin=False):
        """LongestSuffix / ShortestSuffix walked from each string's last byte to its first: length or -1."""
        rev = [bytes(reversed(s)) for s in strings]
        init = np.full(len(strings), self.initial, np.int64)
        if through_end:
            init = self.nxt[init, self.end_cls]
        P, lens, _ = self.paths(rev, init, False)
        out = np.full(len(strings), -1, np.int64)
        for i in range(len(strings)):
            row = P[i, : lens[i] + 1]
            fin, dead = self.final[row], self.dead[row]
            pos, J = -1, int(lens[i])
            for j in range(lens[i] + 1):
                if shortest and (fin[j] or dead[j]) or not shortest and dead[j]:
                    J = j
                    break
            if shortest:
                st = row[J]
                if through_begin:
                    st = self.nxt[st, self.begin_cls]
                if self.final[st]:
                    pos = J
            else:
                hits = np.nonzero(fin[: J + 1])[0]
                if len(hits):
                    pos = int(hits[-1])
                if through_begin and self.final[self.nxt[row[J], self.begin_cls]]:
                    pos = J
            out[i] = pos
        return out

    def match_start(self, text, lo, end, rid, begin_at_lo, end_mark):
        """One reversed walk from ``end`` down to ``lo`` over ``text`` (positions index it), EndMark first when
        ``end_mark``: the least s with rid accepted over [s, end) (rid None: any final state), BeginMark stepped at lo
        when ``begin_at_lo``; the walk stops once rid can no longer be accepted (rid None: in a Dead state).  Returns
        (start or None, open), open meaning the walk reached lo with rid still acceptable and no BeginMark stepped."""
        live = self.live() if rid is not None else None
        st = self.initial
        if end_mark:
            st = self.nxt[st, self.end_cls]

        def ok(s):
            return bool(self.final[s]) and (rid is None or rid in self.accept[s])

        def alive(s):
            return not self.dead[s] if rid is None else bool(live[s, rid])

        best = end if ok(st) else None
        pos = end
        while pos > lo and alive(st):
            pos -= 1
            st = self.nxt[st, self.cls[text[pos]]]
            if ok(st):
                best = pos
        if pos == lo and alive(st):
            if not begin_at_lo:
                return best, True
            if ok(self.nxt[st, self.begin_cls]):
                best = lo
        return best, False

    def match_starts(self, text, wlo, whi, ends, ids, begin, end, max_back=0):
        """MatchStarts for entries (ends, ids; ids None: any final state) in the window [wlo, whi) of text: the
        leftmost start, PIRE_GPU_NO_START (2^64 - 1) for none, and the open flag.  An entry at the window's end under
        ``end`` is walked with and without EndMark, and the longer match wins."""
        starts = np.full(len(ends), 0xFFFFFFFFFFFFFFFF, np.uint64)
        opened = np.zeros(len(ends), np.uint8)
        for k, e in enumerate(np.asarray(ends, np.int64).tolist()):
            lo = e - max_back if max_back and e - wlo > max_back else wlo
            rid = None if ids is None else int(ids[k])
            best, op = None, False
            for em in ((False, True) if end and e == whi else (False,)):
                b, o = self.match_start(text, lo, e, rid, begin and lo == wlo, em)
                op = op or o
                if b is not None and (best is None or b < best):
                    best = b
            if best is not None:
                starts[k] = best
            opened[k] = op
        return starts, opened


def _reach(S, src, dst, seeds):
    """States reachable from ``seeds`` along edges src -> dst."""
    order = np.argsort(src, kind="stable")
    src_s, dst_s = src[order], dst[order]
    begin = np.searchsorted(src_s, np.arange(S + 1))
    seen = np.zeros(S, bool)
    frontier = np.unique(np.asarray(seeds, np.int64))
    seen[frontier] = True
    while len(frontier):
        lo, hi = begin[frontier], begin[frontier + 1]
        cnt = hi - lo
        idx = np.repeat(lo - np.concatenate(([0], np.cumsum(cnt)[:-1])), cnt) + np.arange(int(cnt.sum()))
        nb = np.unique(dst_s[idx])
        frontier = nb[~seen[nb]]
        seen[frontier] = True
    return seen


# ----------------------------------------------------------------------------------------------------- builders

def _partition(rng, L):
    """A random partition of the 256 bytes into L non-empty classes."""
    assert 1 <= L <= 256
    cls = np.concatenate([np.arange(L), rng.integers(0, L, 256 - L)])
    return rng.permutation(cls)


def _table(S, L):
    """An [S, L + 3] table whose byteless column loops and whose other columns are still to be filled."""
    nxt = np.zeros((S, L + 3), np.int64)
    nxt[:, L] = np.arange(S)
    return nxt


def _accepts(rng, final, regexps, max_ids=3):
    acc = []
    for f in final:
        if f and regexps:
            k = int(rng.integers(1, max_ids + 1))
            acc.append(sorted(rng.choice(regexps, size=min(k, regexps), replace=False).tolist()))
        else:
            acc.append([0] if f else [])
    return acc


def uniform(seed, S, L, p, regexps=4):
    """Family 1: a uniform random table of S states over L classes, each state final with probability p."""
    rng = np.random.default_rng(seed)
    nxt = _table(S, L)
    for c in list(range(L)) + [L + 1, L + 2]:
        nxt[:, c] = rng.integers(0, S, S)
    final = rng.random(S) < p if 0 < p < 1 else np.full(S, p >= 1)
    d = Dfa("uniform_S%d_L%d_p%g" % (S, L, p), nxt, _partition(rng, L), final, _accepts(rng, final, regexps),
            int(rng.integers(S)), regexps)
    assert len(np.unique(d.cls)) == L
    assert p <= 0 and not d.final.any() or p >= 1 and d.final.all() or 0 < p < 1
    return d


def hot_edge(seed, reach, extra=6, L=64):
    """Family 2: exactly ``reach`` states reachable over bytes in StaticHotOrder, ``extra`` more that only EndMark
    leads to (or nothing does)."""
    rng = np.random.default_rng(seed)
    S = reach + extra
    nxt = _table(S, L)
    # a random spanning tree over 0..reach-1 from 0 keeps every one of them reachable; other edges stay inside
    for c in range(L):
        nxt[:reach, c] = rng.integers(0, reach, reach)
    for t in range(1, reach):
        nxt[int(rng.integers(0, t)), int(rng.integers(0, L))] = t
    nxt[reach:, :L] = rng.integers(0, reach, (extra, L))
    nxt[:, L + 1] = np.arange(S)
    nxt[0, L + 1] = 0                                             # Begin() stays in the initial state
    nxt[:, L + 2] = rng.integers(0, S, S)
    if extra:
        nxt[1:reach, L + 2] = rng.integers(reach, S, reach - 1)  # EndMark reaches the byte-unreachable rows
    final = rng.random(S) < 0.3
    d = Dfa("hot_reach%d_extra%d" % (reach, extra), nxt, _partition(rng, L), final, _accepts(rng, final, 4), 0, 4)
    order, reached = d.static_hot_order()
    assert reached == reach, (reached, reach)
    return d


def priv_edge(seed, rows):
    """Family 2: exactly ``rows`` hot rows (all states), around PRIV's 47 private rows plus sink and its 115-row
    second tier."""
    d = hot_edge(seed, rows, extra=0)
    _, H, _, _ = d.hot_layout()
    assert H == rows and rows in (PRIV_ROWS - 1, PRIV_ROWS, PRIV_HOT_ROWS, PRIV_HOT_ROWS + 1)
    return d


def look_cold(seed):
    """Family 2: hot id 0 (the first non-final hot row) has a byte to a cold row, so the look-ahead filter is off.
    BeginMark leads to a final row whose 256 distinct children fill the hot rows before the initial row's."""
    rng = np.random.default_rng(seed)
    L = 256
    S = 300
    nxt = _table(S, L)
    nxt[:, :L] = rng.integers(0, S, (S, L))
    B, I = 1, 0
    nxt[I, L + 1] = B
    nxt[:, L + 1] = np.where(np.arange(S) == I, B, np.arange(S))
    nxt[B, :L] = np.arange(2, 2 + L)                             # 256 distinct children, all before I's
    nxt[I, :L] = 270 + rng.integers(0, 30, L)                    # I's children come after them: cold
    nxt[:, L + 2] = rng.integers(0, S, S)
    final = rng.random(S) < 0.2
    final[B], final[I] = True, False
    d = Dfa("look_cold", nxt, np.arange(256), final, _accepts(rng, final, 3), I, 3)
    new, H, ff, look_ok = d.hot_layout()
    assert H == 255 and new[I] == 0 and not look_ok
    return d


def width_edge(seed, S):
    """Family 3: exactly S states, 65 536 (the largest 16-bit table, with id 65 535 in a cell) or 65 537."""
    rng = np.random.default_rng(seed)
    L = 3
    nxt = _table(S, L)
    # a cycle over every state keeps them all reachable and live; the other classes jump anywhere
    perm = rng.permutation(S)
    nxt[perm, 0] = np.roll(perm, -1)
    nxt[:, 1:L] = rng.integers(0, S, (S, L - 1))
    nxt[:, L + 1] = rng.integers(0, S, S)
    nxt[:, L + 2] = rng.integers(0, S, S)
    final = rng.random(S) < 0.05
    d = Dfa("width_%d" % S, nxt, _partition(rng, L), final, _accepts(rng, final, 5), int(perm[0]), 5)
    new, H, _, _ = d.hot_layout()
    old_last = int(np.nonzero(new == S - 1)[0][0])
    assert (d.nxt[:, :L] == old_last).any()                     # the largest id is a transition target
    assert d.states == S
    return d


def shift_register(seed, k, r=3, L=2):
    """Family 4: a delay counter and the last r classes: (min(bytes seen, k), last r classes).  Walks from any two
    states fall together after exactly max(k, r) bytes; finals depend on the remembered classes."""
    rng = np.random.default_rng(seed)
    m = L ** r
    S = (k + 1) * m
    nxt = _table(S, L)
    cnt, hist = np.divmod(np.arange(S), m)
    for c in range(L):
        nxt[:, c] = np.minimum(cnt + 1, k) * m + (hist * L + c) % m
    nxt[:, L + 1] = np.arange(S)
    nxt[:, L + 2] = np.arange(S)
    fin_hist = rng.random(m) < 0.4
    final = (cnt == k) & fin_hist[hist]
    d = Dfa("shift_k%d" % k, nxt, _partition(rng, L), final, _accepts(rng, final, 2), 0, 2)
    assert convergence(d, max(k, r) + 2, rng) == max(k, r)
    return d


def permutation(seed, S=5, L=3):
    """Family 4: every class permutes the states, so walks from different states never fall together."""
    rng = np.random.default_rng(seed)
    nxt = _table(S, L)
    for c in range(L):
        nxt[:, c] = rng.permutation(S)
    nxt[:, L + 1] = rng.permutation(S)
    nxt[:, L + 2] = rng.permutation(S)
    final = np.zeros(S, bool)
    final[rng.choice(S, size=2, replace=False)] = True
    d = Dfa("perm_S%d" % S, nxt, _partition(rng, L), final, _accepts(rng, final, 2), 0, 2)
    assert convergence(d, 64, rng) is None
    return d


def convergence(d, limit, rng):
    """The number of bytes after which the walks from all states coincide on a random string, or None."""
    cur = np.arange(d.states)
    text = rng.integers(0, 256, limit)
    for j in range(limit):
        if len(np.unique(cur)) == 1:
            return j
        cur = d.nxt[cur, d.cls[text[j]]]
    return None if len(np.unique(cur)) > 1 else limit


def marks(seed):
    """Family 5: BeginMark and EndMark lead to rows no byte reaches; rows final only after EndMark; ids that only
    EndMark still makes acceptable (the ``live`` table must propagate over the marks)."""
    rng = np.random.default_rng(seed)
    L, core, side = 8, 24, 8
    S = core + 2 * side
    nxt = _table(S, L)
    nxt[:core, :L] = rng.integers(0, core, (core, L))
    nxt[core:core + side, :L] = rng.integers(core, core + side, (side, L))   # each side keeps to itself over bytes
    nxt[core + side:, :L] = rng.integers(core + side, S, (side, L))
    nxt[:, L + 1] = np.where(np.arange(S) < core, core + rng.integers(0, side, S), np.arange(S))
    nxt[:, L + 2] = np.where(np.arange(S) < core, core + side + rng.integers(0, side, S), np.arange(S))
    final = np.zeros(S, bool)
    final[core + side:] = True                                   # final only behind EndMark
    final[core: core + side] = rng.random(side) < 0.5            # behind BeginMark, some
    acc = [[] for _ in range(S)]
    for s in range(core, S):
        if final[s]:
            acc[s] = [int(x) for x in rng.choice(6, size=2, replace=False)]
    acc[S - 1] = [5]                                             # id 5 only behind EndMark, reached by EndMark only
    for s in range(core + side, S - 1):
        acc[s] = [i for i in acc[s] if i != 5] or [0]
    d = Dfa("marks", nxt, _partition(rng, L), final, acc, 0, 6)
    _, reached = d.static_hot_order()
    assert reached <= core + side and not d.final[:core].any()
    live = d.live()
    assert live[:core, 5].any()                                  # id 5 acceptable from a byte row, through EndMark only
    return d


def absorbing(seed, early):
    """Family 6: an absorbing final row (NoExit) reached within a few bytes (``early``) or only after a long chain."""
    rng = np.random.default_rng(seed)
    L, chain = 4, (3 if early else 300)
    S = chain + 2
    nxt = _table(S, L)
    for c in range(L):
        nxt[:chain, c] = np.arange(1, chain + 1) if c == 0 else rng.integers(0, chain, chain)
    nxt[chain, :L] = chain                                       # absorbing final
    nxt[chain + 1, :L] = rng.integers(0, chain, L)
    nxt[:, L + 1] = np.arange(S)
    nxt[:, L + 2] = np.arange(S)
    nxt[0, L + 2] = chain + 1
    final = np.zeros(S, bool)
    final[chain] = True
    final[chain + 1] = True
    cls = np.zeros(256, np.int64)
    cls[rng.choice(256, size=3 * 64, replace=False)] = rng.integers(1, L, 3 * 64)
    d = Dfa("absorb_%s" % ("early" if early else "late"), nxt, cls, final, _accepts(rng, final, 2), 0, 2)
    m0, _ = d._exit_masks()
    assert m0[chain] == NO_EXIT
    return d


def counting(seed, regexps, times=1, absorbing_initial=False, S=40, L=16):
    """Family 7: counting images.  Final rows list ids ``times`` times each (15 stays packed, 16 falls back to the
    lists); with ``absorbing_initial`` the initial row is final, absorbing and lists every id ``times`` times, so that
    Initialize, BeginMark and every byte add ``times`` to each counter."""
    rng = np.random.default_rng(seed)
    nxt = _table(S, L)
    nxt[:, :L] = rng.integers(0, S, (S, L))
    nxt[:, L + 1] = rng.integers(0, S, S)
    nxt[:, L + 2] = rng.integers(0, S, S)
    final = rng.random(S) < 0.4
    acc = []
    for s in range(S):
        if final[s]:
            ids = sorted(rng.choice(regexps, size=min(regexps, int(rng.integers(1, 4))), replace=False).tolist())
            acc.append([i for i in ids for _ in range(times)])
        else:
            acc.append([])
    initial = 0
    if absorbing_initial:
        nxt[0, :] = 0
        nxt[0, L] = 0
        final[0] = True
        acc[0] = [i for i in range(regexps) for _ in range(times)]
    else:
        final[0] = False
        acc[0] = []
    d = Dfa("count_r%d_x%d%s" % (regexps, times, "_abs" if absorbing_initial else ""), nxt, _partition(rng, L), final, acc,
            initial, regexps)
    most = max((max(a.count(i) for i in set(a)) for a in acc if a), default=0)
    assert most == times, (most, times)
    return d


def newline_class(seed, S=30, L=12):
    """A uniform table in which '\\n' has a class of its own (for line batches)."""
    d = uniform(seed, S, L, 0.3)
    cls = d.cls.copy()
    cls[cls == L - 1] = 0
    cls[ord("\n")] = L - 1
    out = Dfa("lines_S%d" % S, d.nxt, cls, d.final, d.accept, d.initial, d.regexps)
    assert (out.cls == out.cls[10]).sum() == 1
    return out


# The families by name: each entry builds one automaton from a fixed seed.
FAMILIES = {
    "uniform_L1": lambda: uniform(11, 17, 1, 0.3),
    "uniform_L2": lambda: uniform(12, 40, 2, 0.3),
    "uniform_L200": lambda: uniform(13, 300, 200, 0.2),
    "uniform_L256": lambda: uniform(14, 64, 256, 0.1),
    "uniform_p0": lambda: uniform(15, 50, 10, 0.0),
    "uniform_p1": lambda: uniform(16, 50, 10, 1.0),
    "hot_254": lambda: hot_edge(21, 254),
    "hot_255": lambda: hot_edge(22, 255),
    "hot_256": lambda: hot_edge(23, 256),
    "priv_47": lambda: priv_edge(24, 47),
    "priv_48": lambda: priv_edge(25, 48),
    "priv_115": lambda: priv_edge(26, 115),
    "priv_116": lambda: priv_edge(27, 116),
    "look_cold": lambda: look_cold(28),
    "width_65536": lambda: width_edge(31, 65536),
    "width_65537": lambda: width_edge(32, 65537),
    "shift_16": lambda: shift_register(41, 16),
    "shift_33": lambda: shift_register(42, 33),
    "shift_64": lambda: shift_register(43, 64),
    "perm_5": lambda: permutation(44),
    "marks": lambda: marks(51),
    "absorb_early": lambda: absorbing(61, True),
    "absorb_late": lambda: absorbing(62, False),
    "count_r1": lambda: counting(71, 1),
    "count_r8_x15": lambda: counting(72, 8, 15),
    "count_r9": lambda: counting(73, 9, 2),
    "count_r16_x15": lambda: counting(74, 16, 15),
    "count_r16_x16": lambda: counting(75, 16, 16),
    "count_r17": lambda: counting(76, 17, 3),
    "count_r33": lambda: counting(77, 33),
    "count_r257": lambda: counting(78, 257, 2, S=60),
    "count_abs16_x15": lambda: counting(79, 16, 15, absorbing_initial=True),
    "lines": lambda: newline_class(81),
}

_CACHE = {}


def family(name):
    """The automaton of one family (built once per process)."""
    if name not in _CACHE:
        _CACHE[name] = FAMILIES[name]()
    return _CACHE[name]
