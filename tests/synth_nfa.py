"""Seeded random NFAs written as Pire::SlowScanner images, and a numpy bit-set walker as their oracle.

The reference's front end only makes the NFAs its patterns need; these reach the shapes the SlowScanner kernels branch
on: every set width (S = 1 .. 4096, one to 128 words, both sides of the lane/warp boundary at 256), up to 264 letters,
empty and dense jump lists, duplicate jumps, and S = 4097 for the refusal.

The image is what SlowScanner::Save() writes (pire/scanner_io.cpp:71-110): the 24-byte header with type 3, Locals
{statesCount, lettersCount, start}, the empty flag padded to 8, size_t letters[264], bool finals[S] padded to 8,
size_t jumpPos[S * L + 1], unsigned jumps[] padded to 8.
"""
import struct

import numpy as np

MAX_CHAR = 264
EPSILON, BEGIN_MARK, END_MARK = 257, 258, 259


def _pad8(b):
    return b + b"\0" * (-len(b) % 8)


class SynthNfa:
    """states, letters, start; letter_of[264]; finals[S] bool; jumps[s][l] = list of targets (duplicates allowed)."""

    def __init__(self, states, letters, start, letter_of, finals, jumps):
        self.states, self.letters, self.start = states, letters, start
        self.letter_of = np.asarray(letter_of, np.int64)
        self.finals = np.asarray(finals, bool)
        self.jumps = jumps
        self.words = (states + 31) // 32
        # succ[l, s] = successor set of s on l as a bool row
        self.succ = np.zeros((letters, states, states), bool)
        for s in range(states):
            for l in range(letters):
                for t in jumps[s][l]:
                    self.succ[l, s, t] = True

    def image(self, empty=False):
        out = struct.pack("<6I", 0x45524950, 7, 8, 16, 3, 24)
        out += struct.pack("<3Q", self.states, self.letters, self.start)
        out += _pad8(struct.pack("<?", empty))
        if empty:
            return out
        out += struct.pack("<%dQ" % MAX_CHAR, *[int(x) for x in self.letter_of])
        out += _pad8(bytes(int(f) for f in self.finals))
        pos, flat = [0], []
        for s in range(self.states):
            for l in range(self.letters):
                flat += self.jumps[s][l]
                pos.append(len(flat))
        out += struct.pack("<%dQ" % len(pos), *pos)
        out += _pad8(struct.pack("<%dI" % len(flat), *flat))
        return out

    # --- oracle: sets as bool vectors, packed to u32 words ---------------------------------------------
    def initial(self):
        v = np.zeros(self.states, bool)
        v[self.start] = True
        return v

    def step(self, cur, symbol):
        l = self.letter_of[symbol]
        return self.succ[l][cur].any(axis=0) if cur.any() else np.zeros(self.states, bool)

    def final(self, cur):
        return bool((cur & self.finals).any())

    def pack(self, cur):
        bits = np.zeros(self.words * 32, bool)
        bits[: self.states] = cur
        return np.packbits(bits, bitorder="little").view(np.uint32)

    def unpack(self, words):
        bits = np.unpackbits(np.asarray(words, np.uint32).view(np.uint8), bitorder="little")
        return bits[: self.states].astype(bool)

    def run(self, data, start=None, begin=True, end=True):
        """Runner(sc[, st]) [.Begin()] .Run(data) [.End()]: (Final(), the packed set)."""
        cur = self.initial() if start is None else start
        if begin:
            cur = self.step(cur, BEGIN_MARK)
        for b in data:
            if not cur.any():
                break
            cur = self.step(cur, b)
        if end:
            cur = self.step(cur, END_MARK)
        return self.final(cur), self.pack(cur)


def random_nfa(seed, states, letters, density=2.0, final_share=0.1, dup_share=0.0, empty_share=0.0):
    """A random NFA: every (state, letter) has about `density` jumps (none with probability `empty_share`), a share of
    them listed twice; bytes and marks map to random letters."""
    rng = np.random.default_rng(seed)
    letter_of = rng.integers(0, letters, MAX_CHAR)
    letter_of[EPSILON] = 0
    letter_of[260:] = 0
    finals = rng.random(states) < final_share
    start = int(rng.integers(0, states))
    jumps = []
    for s in range(states):
        row = []
        for l in range(letters):
            if rng.random() < empty_share:
                row.append([])
                continue
            k = int(rng.poisson(density))
            t = [int(x) for x in rng.integers(0, states, k)]
            t += [x for x in t if rng.random() < dup_share]
            row.append(t)
        jumps.append(row)
    return SynthNfa(states, letters, start, letter_of, finals, jumps)


# The families the tests run: (name, seed, states, letters, density, final share, duplicate share, empty share).
FAMILIES = [
    ("s1", 1, 1, 3, 1.0, 0.5, 0.5, 0.2),
    ("s31", 2, 31, 8, 1.5, 0.1, 0.2, 0.3),
    ("s32", 3, 32, 4, 1.2, 0.1, 0.0, 0.2),
    ("s33", 4, 33, 16, 1.2, 0.1, 0.3, 0.2),
    ("s64_l264", 5, 64, 264, 1.0, 0.1, 0.1, 0.3),
    ("s100", 6, 100, 6, 1.5, 0.05, 0.2, 0.2),
    ("s255_dense", 7, 255, 5, 20.0, 0.05, 0.3, 0.0),
    ("s256", 8, 256, 4, 1.2, 0.05, 0.1, 0.2),
    ("s257", 9, 257, 4, 1.2, 0.05, 0.1, 0.2),
    ("s700", 10, 700, 7, 1.1, 0.02, 0.1, 0.3),
    ("s1024", 11, 1024, 3, 1.1, 0.02, 0.1, 0.3),
    ("s1500", 12, 1500, 3, 1.0, 0.02, 0.1, 0.3),
    ("s4096", 13, 4096, 2, 1.0, 0.01, 0.05, 0.3),
]


def family(name):
    for f in FAMILIES:
        if f[0] == name:
            return random_nfa(f[1], f[2], f[3], f[4], f[5], f[6], f[7])
    raise KeyError(name)
