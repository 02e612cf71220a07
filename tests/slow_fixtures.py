"""The SlowScanner fixtures of tests/golden/slow_images.json.xz (written by tests/golden/make_slow_images.py from the
reference), decoded."""
import base64
import json
import lzma
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


class SlowEntry:
    def __init__(self, d):
        self.name = d["name"]
        self.image = lzma.decompress(base64.b64decode(d["image"]))
        self.states, self.letters, self.empty = d["states"], d["letters"], d["empty"]
        self.determinable = d["determinable"]
        self.words = (self.states + 31) // 32
        self.strings = [bytes.fromhex(s) for s in d["strings"]]
        self.start_sets = np.frombuffer(bytes.fromhex(d["start_sets"]), np.uint32).reshape(len(self.strings), self.words)
        # (begin, end, from_sets) -> (final bool[n], sets uint32[n, words])
        self.runs = {}
        for r in d["runs"]:
            sets = np.frombuffer(bytes.fromhex(r["sets"]), np.uint32).reshape(len(self.strings), self.words)
            self.runs[(r["begin"], r["end"], r["from_sets"])] = (np.array(r["final"], bool), sets)

    def __repr__(self):
        return "SlowEntry(%s)" % self.name


def load():
    with open(os.path.join(HERE, "golden", "slow_images.json.xz"), "rb") as f:
        return [SlowEntry(e) for e in json.loads(lzma.decompress(f.read()))["entries"]]


SLOW = load()
