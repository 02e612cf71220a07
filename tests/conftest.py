import base64
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")


class GoldenCase:
    def __init__(self, d):
        self.name = d["name"]
        self.patterns = [(bytes.fromhex(p), o) for p, o in d["patterns"]]
        self.image = base64.b64decode(d["image"])
        self.strings = [bytes.fromhex(s) for s in d["strings"]]
        self.final = d["final"]
        self.ids = d["ids"]
        self.state = d["state"]
        self.begin = bool(d["begin"])
        self.end = bool(d["end"])
        self.states, self.letters, self.regexps = d["states"], d["letters"], d["regexps"]

    def mask(self):
        return [sum(1 << i for i in ids if i < 32) for ids in self.ids]

    def __repr__(self):
        return "GoldenCase(%s)" % self.name


def load_golden():
    with open(os.path.join(HERE, "golden", "pire_golden.json")) as f:
        return [GoldenCase(c) for c in json.load(f)["cases"]]


def load_golden_prefix():
    with open(os.path.join(HERE, "golden", "pire_golden.json")) as f:
        return [(bytes.fromhex(c["pattern"]), base64.b64decode(c["image"]), bytes.fromhex(c["text"]), c["shortest"], c["longest"])
                for c in json.load(f)["prefix_cases"]]


class CountCase:
    """count_ut.cpp HalfFinal@553: the glue of the five HalfFinalFsm counters of one pattern."""

    def __init__(self, d):
        import lzma
        self.pattern = bytes.fromhex(d["pattern"])
        self.image = lzma.decompress(base64.b64decode(d["image_xz"]))
        self.strings = [bytes.fromhex(s) for s in d["strings"]]
        self.counts, self.final, self.expect = d["counts"], d["final"], d["expect"]
        self.states, self.regexps = d["states"], d["regexps"]
        self.single = None
        if "single" in d:
            self.single = (lzma.decompress(base64.b64decode(d["single"]["image_xz"])), d["single"]["counts"], d["single"]["final"])

    def __repr__(self):
        return "CountCase(%r, %r)" % (self.pattern, self.strings[0])


def load_golden_counts():
    with open(os.path.join(HERE, "golden", "pire_golden.json")) as f:
        return [CountCase(c) for c in json.load(f)["count_cases"]]


def load_golden_suffix():
    with open(os.path.join(HERE, "golden", "pire_golden.json")) as f:
        return [(bytes.fromhex(c["pattern"]), base64.b64decode(c["image"]), [bytes.fromhex(t) for t in c["texts"]], c["shortest"],
                 c["longest"]) for c in json.load(f)["suffix_cases"]]


GOLDEN = load_golden()
GOLDEN_SUFFIX = load_golden_suffix()
GOLDEN_COUNTS = load_golden_counts()
GOLDEN_PREFIX = load_golden_prefix()


@pytest.fixture(scope="session")
def golden():
    return GOLDEN


@pytest.fixture(scope="session")
def ref():
    """The reference: the real one when oracle/_ref is built, else its answers stored under tests/golden (see
    refpire.StoredRef).  PIRE_RECORD_REFERENCE=<file> records what the session asks of the real one into <file>."""
    import refpire
    record = os.environ.get("PIRE_RECORD_REFERENCE")
    if not refpire.have_ref():
        if record:
            pytest.fail("PIRE_RECORD_REFERENCE needs oracle/_ref (oracle/build_ref.sh)")
        yield refpire.StoredRef()
        return
    if not record:
        yield refpire.Ref()
        return
    recorder = refpire.StoredRef(live=refpire.Ref())
    yield recorder
    recorder.store.save(record)


@pytest.fixture(scope="session")
def cuda_device():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("this test is marked gpu but no CUDA device is visible")
    return 0
