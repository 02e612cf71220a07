"""Python mirror of the reference's Scanner / Runner / Matches surface for the
batch scan path, over the C ABI (include/pire_b200.h).

Reference interface mirrored (same names and argument meaning):
    Pire::Scanner             Size / Empty / RegexpsCount / LettersCount /
                              Initialize / Next / Final / Dead / AcceptedRegexps /
                              StateIndex / Load          pire/scanners/multi.h:134-194,:244-311
    Pire::Runner(sc)          .Begin().Run(...).End()    pire/run.h:365-392
    Pire::Matches(sc, ...)    no Begin/End marks         pire/run.h:396-400

The one difference is the unit of work: Run() takes a *batch* of strings
resident in HBM (``Batch``) instead of one ``const char*`` range, and the
RunHelper answers per string.  torch is used only to own device memory and to
name the CUDA stream.
"""
import ctypes as C

import numpy as np

from . import _native as N

BeginMark = 258   # pire/defs.h:63
EndMark = 259     # pire/defs.h:64


def _torch():
    import torch
    return torch


class Batch:
    """A batch of strings on one GPU: ``corpus`` (uint8 CUDA tensor) plus either CSR
    ``offsets`` (int64/uint64 CUDA tensor, n+1 entries) or a fixed string length."""

    def __init__(self, corpus, offsets=None, fixed_len=0, n=None):
        torch = _torch()
        if corpus.dtype != torch.uint8 or not corpus.is_cuda or not corpus.is_contiguous():
            raise ValueError("corpus must be a contiguous uint8 CUDA tensor")
        self.corpus = corpus
        self.offsets = offsets
        self.fixed_len = int(fixed_len)
        if offsets is not None:
            if offsets.dtype not in (torch.int64, torch.uint64) or not offsets.is_cuda or not offsets.is_contiguous():
                raise ValueError("offsets must be a contiguous int64 CUDA tensor")
            self.n = offsets.numel() - 1 if n is None else int(n)
        else:
            if n is None:
                n = corpus.numel() // self.fixed_len if self.fixed_len else 0
            self.n = int(n)
            if self.n * self.fixed_len > corpus.numel():
                raise ValueError("corpus shorter than n * fixed_len")
        self.device = corpus.device
        self.order = None          # set by bin_by_length()
        self.trim = 0              # 1 for line batches (from_text): the newline ending a line is not part of it

    def bin_by_length(self):
        """Sort the strings by descending length (on the device) so that the lanes of a warp
        scan strings of similar length; results stay indexed by the original string number."""
        torch = _torch()
        if self.offsets is None or self.n == 0:
            return self
        order = torch.empty(self.n, dtype=torch.int32, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        N.check(N.lib.pire_gpu_length_order(self.offsets.data_ptr(), self.n, order.data_ptr(), self.device.index or 0, stream),
                "pire_gpu_length_order")
        self.order = order
        return self

    @classmethod
    def from_text(cls, text):
        """Lines of a newline-delimited text (uint8 CUDA tensor), found on the device with
        std::getline semantics -- what samples/pigrep/pigrep.cpp:38-45 feeds to Runner per line."""
        torch = _torch()
        if text.dtype != torch.uint8 or not text.is_cuda or not text.is_contiguous():
            raise ValueError("text must be a contiguous uint8 CUDA tensor")
        dev = text.device
        stream = torch.cuda.current_stream(dev).cuda_stream
        n_lines = C.c_uint64(0)
        cap = max(1024, text.numel() // 64)
        while True:
            offsets = torch.empty(cap + 1, dtype=torch.int64, device=dev)
            rc = N.lib.pire_gpu_split_lines(text.data_ptr(), text.numel(), offsets.data_ptr(), cap, C.byref(n_lines),
                                            dev.index or 0, stream)
            if rc == 0:
                break
            if rc == -1 and n_lines.value > cap:         # buffer too small: retry with the reported capacity
                cap = int(n_lines.value)
                continue
            N.check(rc, "pire_gpu_split_lines")
        b = cls(text, offsets[: n_lines.value + 1].contiguous(), n=int(n_lines.value))
        b.trim = 1
        return b

    @classmethod
    def from_strings(cls, strings, device="cuda:0"):
        """Host convenience: pack Python byte strings (CSR) and upload."""
        torch = _torch()
        offs = np.zeros(len(strings) + 1, np.int64)
        np.cumsum([len(s) for s in strings], out=offs[1:])
        blob = np.frombuffer(b"".join(strings) + b"\0" * 32, dtype=np.uint8).copy()
        return cls(torch.from_numpy(blob).to(device), torch.from_numpy(offs).to(device), n=len(strings))

    def payload_bytes(self):
        if self.offsets is None:
            return self.n * self.fixed_len
        o = self.offsets
        return int(o[self.n].item() - o[0].item()) - self.trim * self.n


class Scanner:
    """A compiled multi-regexp scanner resident on one GPU (Pire::Scanner's role)."""

    def __init__(self, image, device=0):
        image = bytes(image)
        h = C.c_void_p()
        buf = (C.c_char * len(image)).from_buffer_copy(image)
        N.check(N.lib.pire_gpu_scanner_create(buf, len(image), int(device), C.byref(h)), "pire_gpu_scanner_create")
        self._h = h
        self.device = int(device)

    # Scanner::Load(yistream*) -- multi.h:575-599
    @classmethod
    def Load(cls, image, device=0):
        return cls(image, device)

    def __del__(self):
        h = getattr(self, "_h", None)
        lib = getattr(N, "lib", None)          # None while the interpreter is shutting down
        if h and lib is not None:
            lib.pire_gpu_scanner_destroy(h)
            self._h = None

    def info(self):
        out = N.Info()
        N.check(N.lib.pire_gpu_scanner_info(self._h, C.byref(out)), "pire_gpu_scanner_info")
        return out

    def Size(self):
        return self.info().states

    def Empty(self):
        return bool(self.info().empty)

    def set_count_mode(self, mode):
        """0 auto, 1 accept lists, 2 packed increments, 3 packed on every chunk (pire_gpu_scanner_set_count_mode)."""
        N.check(N.lib.pire_gpu_scanner_set_count_mode(self._h, mode), "pire_gpu_scanner_set_count_mode")

    def RegexpsCount(self):
        return self.info().regexps

    def LettersCount(self):
        return self.info().letters

    # --- host-side Scanner concept (index space) ------------------------------
    def Initialize(self):
        return N.lib.pire_gpu_initial(self._h)

    def Next(self, state, ch):
        return N.lib.pire_gpu_next(self._h, state, ch)

    def Final(self, state):
        return bool(N.lib.pire_gpu_final(self._h, state))

    def Dead(self, state):
        return bool(N.lib.pire_gpu_dead(self._h, state))

    def AcceptedRegexps(self, state):
        ids = (C.c_uint32 * 1024)()
        k = N.lib.pire_gpu_accepted_regexps(self._h, state, ids, 1024)
        return [int(ids[i]) for i in range(min(k, 1024))]

    @staticmethod
    def StateIndex(state):
        return state

    # --- device ------------------------------------------------------------------
    def set_variant(self, variant):
        N.check(N.lib.pire_gpu_scanner_set_variant(self._h, variant), "pire_gpu_scanner_set_variant")

    def set_max_hot(self, rows):
        N.check(N.lib.pire_gpu_scanner_set_max_hot(self._h, rows), "pire_gpu_scanner_set_max_hot")

    def Tune(self, batch, n_sample=None, begin=True, end=True):
        """Pick the shared-memory rows from the states a sample of `batch` visits."""
        n_sample = batch.n if n_sample is None else min(int(n_sample), batch.n)
        flags = (N.RUN_BEGIN if begin else 0) | (N.RUN_END if end else 0) | (N.RUN_LINES if batch.trim else 0)
        torch = _torch()
        stream = torch.cuda.current_stream(batch.device).cuda_stream
        N.check(N.lib.pire_gpu_scanner_tune(self._h, batch.corpus.data_ptr(),
                                            batch.offsets.data_ptr() if batch.offsets is not None else None,
                                            batch.fixed_len, n_sample, flags, stream), "pire_gpu_scanner_tune")

    def AutoSelect(self, batch, begin=True, end=True):
        """Time the kernel variants on `batch` and keep the fastest as the AUTO choice.
        Returns {variant name: ms}."""
        flags = (N.RUN_BEGIN if begin else 0) | (N.RUN_END if end else 0) | (N.RUN_LINES if batch.trim else 0)
        torch = _torch()
        stream = torch.cuda.current_stream(batch.device).cuda_stream
        ms = (C.c_float * N.VARIANT_SLOTS)()
        N.check(N.lib.pire_gpu_scanner_autoselect(self._h, batch.corpus.data_ptr(),
                                                  batch.offsets.data_ptr() if batch.offsets is not None else None,
                                                  batch.fixed_len, batch.n, flags, stream, ms),
                "pire_gpu_scanner_autoselect")
        return {name: float(ms[v]) for v, name in N.VARIANT_NAMES.items() if ms[v] > 0}

    def run_batch(self, batch, flags, match_bits=None, accept_masks=None, state_idx=None, stream=None, start_idx=None):
        """Thin wrapper of pire_gpu_run_batch: asynchronous on the current stream.  ``start_idx`` (an int32 CUDA tensor of
        n StateIndex values, reference numbering) starts string i from start_idx[i] (pire_gpu_run_batch_from, ``Runner(sc,
        st)`` per string); it may be ``state_idx`` itself, so that rounds of a batch of streams chain in place."""
        torch = _torch()
        if stream is None:
            stream = torch.cuda.current_stream(batch.device).cuda_stream
        ptr = lambda t: None if t is None else t.data_ptr()
        if start_idx is not None:
            if getattr(batch, "trim", 0):
                raise ValueError("line batches have no per-string starts")
            if start_idx.dtype != torch.int32 or not start_idx.is_cuda or not start_idx.is_contiguous() \
                    or start_idx.numel() < batch.n:
                raise ValueError("start_idx must be a contiguous int32 CUDA tensor of n states")
            order = getattr(batch, "order", None)
            N.check(N.lib.pire_gpu_run_batch_from(self._h, batch.corpus.data_ptr(), ptr(batch.offsets), ptr(order), batch.fixed_len,
                                                  batch.n, flags, start_idx.data_ptr(), ptr(match_bits), ptr(accept_masks),
                                                  ptr(state_idx), stream),
                    "pire_gpu_run_batch_from")
            return
        if getattr(batch, "trim", 0):
            order = batch.order.data_ptr() if batch.order is not None else None
            N.check(N.lib.pire_gpu_run_lines(self._h, batch.corpus.data_ptr(), ptr(batch.offsets), order, batch.n, flags,
                                             ptr(match_bits), ptr(accept_masks), ptr(state_idx), stream),
                    "pire_gpu_run_lines")
            return
        if getattr(batch, "order", None) is not None:
            N.check(N.lib.pire_gpu_run_batch_ordered(self._h, batch.corpus.data_ptr(), ptr(batch.offsets),
                                                     batch.order.data_ptr(), batch.n, flags, ptr(match_bits),
                                                     ptr(accept_masks), ptr(state_idx), stream),
                    "pire_gpu_run_batch_ordered")
            return
        N.check(N.lib.pire_gpu_run_batch(self._h, batch.corpus.data_ptr(), ptr(batch.offsets), batch.fixed_len,
                                         batch.n, flags, ptr(match_bits), ptr(accept_masks), ptr(state_idx), stream),
                "pire_gpu_run_batch")

    def run_batch_host(self, corpus, offsets=None, fixed_len=0, n=None, flags=N.RUN_BEGIN | N.RUN_END,
                       want_masks=False, want_states=False):
        """Host buffers in, host results out (pire_gpu_run_batch_host): numpy arrays
        (or pinned torch CPU tensors viewed as numpy)."""
        corpus = np.ascontiguousarray(corpus, dtype=np.uint8)
        if offsets is not None:
            offsets = np.ascontiguousarray(offsets).view(np.uint64)
            n = len(offsets) - 1 if n is None else n
        elif n is None:
            n = len(corpus) // fixed_len if fixed_len else 0
        bits = np.zeros((n + 31) // 32, np.uint32)
        masks = np.zeros(n, np.uint32) if want_masks else None
        states = np.zeros(n, np.uint32) if want_states else None
        p = lambda a: None if a is None else a.ctypes.data
        N.check(N.lib.pire_gpu_run_batch_host(self._h, p(corpus), corpus.nbytes, p(offsets), fixed_len, n, flags,
                                              p(bits), p(masks), p(states)), "pire_gpu_run_batch_host")
        return bits, masks, states


class RunHelper:
    """Pire::RunHelper (run.h:365-386) over a batch.  ``Begin()`` / ``End()`` record the
    mark steps, ``Run(batch)`` names the strings; the single fused launch happens when
    a result is first asked for.

    ``states`` (an int32 CUDA tensor of n StateIndex values) starts every string from its own state: ``Runner(sc, st)``
    (run.h:391-392) for each string.  ``StateTensor()`` hands the states reached to the next round without a synchronise,
    so a batch of streams arriving in pieces chains as ``prev = Runner(sc, prev.StateTensor()).Run(next_pieces)``."""

    def __init__(self, sc, states=None):
        self.Sc = sc
        self._start = states
        self._begin = False
        self._end = False
        self._batch = None
        self._bits = self._masks = self._states = None

    def Begin(self):
        if self._batch is not None:
            raise ValueError("Begin() must precede Run()")
        self._begin = True
        return self

    def Run(self, batch):
        if self._batch is not None:
            raise ValueError("one Run() per RunHelper on the batch path")
        self._batch = batch
        return self

    def End(self):
        self._end = True
        return self

    def _launch(self):
        if self._bits is not None:
            return
        if self._batch is None:
            raise ValueError("Run() was not called")
        torch = _torch()
        b = self._batch
        dev = b.device
        self._bits = torch.empty((b.n + 31) // 32, dtype=torch.int32, device=dev)
        self._masks = torch.empty(b.n, dtype=torch.int32, device=dev)
        self._states = torch.empty(b.n, dtype=torch.int32, device=dev)
        flags = (N.RUN_BEGIN if self._begin else 0) | (N.RUN_END if self._end else 0)
        self.Sc.run_batch(b, flags, self._bits, self._masks, self._states, start_idx=self._start)

    # per-string results -------------------------------------------------------------
    def StateTensor(self):
        """The device tensor (int32, n) of the states reached, reference numbering, without a synchronise: the
        ``states`` of the next round's Runner."""
        self._launch()
        return self._states

    def MatchBits(self):
        """Packed device bitmap: bit i%32 of word i/32 = Final() of string i."""
        self._launch()
        return self._bits

    def Matches(self):
        """numpy bool[n]: RunHelper::operator bool (run.h:380-381) per string."""
        self._launch()
        words = self._bits.cpu().numpy().view(np.uint32)
        bits = np.unpackbits(words.view(np.uint8), bitorder="little")
        return bits[: self._batch.n].astype(bool)

    def AcceptMasks(self):
        self._launch()
        return self._masks.cpu().numpy().view(np.uint32)

    def States(self):
        """StateIndex() of each string's last state (reference numbering)."""
        self._launch()
        return self._states.cpu().numpy().view(np.uint32)

    def AcceptedRegexps(self, i):
        """Scanner::AcceptedRegexps(State()) for string i (multi.h:149-158)."""
        return self.Sc.AcceptedRegexps(int(self.States()[i]))


class StringRunner:
    """Pire::RunHelper (run.h:365-392) for ONE string resident in HBM, scanned by the whole GPU
    (pire_gpu_run_string).  ``Run(text)`` may be called many times: the texts are scanned as one string, the state
    carried from call to call in a device word, so chained calls do not synchronise (a stream arriving in chunks).
    ``state`` = a StateIndex to start from (``Runner(sc, st)``, run.h:391-392), None = Initialize().  Every ``Run()``
    launches at once on the current stream, so a buffer may be refilled behind it in stream order; ``Begin()`` is
    folded into the first launch, ``End()`` is a launch of its own.  Results (``State()``, ``Final()``,
    ``AcceptedRegexps()``, ``bool``) synchronise.

    To tune the shared-memory rows for a long string, pass a fixed-length view of it to ``Scanner.Tune``, e.g.
    ``sc.Tune(Batch(text[: len(text) // 4096 * 4096], fixed_len=4096))``."""

    def __init__(self, sc, state=None):
        self.Sc = sc
        self._start = None if state is None else int(state)
        self._words = None         # device: [StateIndex, match word, accept mask]
        self._begin = False
        self._ran = False          # a launch has written the state word

    def Begin(self):
        if self._ran:
            raise ValueError("Begin() must precede Run()")
        self._begin = True
        return self

    def Run(self, text):
        torch = _torch()
        if text.dtype != torch.uint8 or not text.is_cuda or not text.is_contiguous() or text.device.index != self.Sc.device:
            raise ValueError("text must be a contiguous uint8 CUDA tensor on the scanner's device")
        self._launch(text, 0)
        return self

    def End(self):
        self._launch(None, N.RUN_END)
        return self

    def _launch(self, text, flags):
        if self._begin:
            flags |= N.RUN_BEGIN
            self._begin = False
        start = stream = None
        if self.Sc.device >= 0:
            torch = _torch()
            dev = torch.device("cuda", self.Sc.device)
            if self._words is None:
                self._words = torch.empty(3, dtype=torch.int32, device=dev)
                if self._start is not None:
                    word = self._start & 0xFFFFFFFF
                    self._words[0] = word - (1 << 32) if word >= (1 << 31) else word
            stream = torch.cuda.current_stream(dev).cuda_stream
            if self._ran or self._start is not None:
                start = self._words.data_ptr()
        ptr = None if self._words is None else self._words.data_ptr()
        N.check(N.lib.pire_gpu_run_string(self.Sc._h, None if text is None else text.data_ptr(), 0 if text is None else text.numel(),
                                          flags, start, None if ptr is None else ptr + 4, None if ptr is None else ptr + 8, ptr,
                                          stream), "pire_gpu_run_string")
        self._ran = True

    def _results(self):
        if not self._ran:
            self._launch(None, 0)          # nothing run yet: the start state itself (after Begin() if it was asked for)
        return self._words.cpu().numpy().view(np.uint32)

    def State(self):
        """StateIndex() of the state reached (reference numbering); 0xFFFFFFFF for a start outside the scanner."""
        return int(self._results()[0])

    def Final(self):
        return bool(self._results()[1] & 1)

    def __bool__(self):
        return self.Final()

    def AcceptMask(self):
        """AcceptedRegexps as a bit mask of the ids below 32."""
        return int(self._results()[2])

    def AcceptedRegexps(self):
        return self.Sc.AcceptedRegexps(self.State())


class StringCounter:
    """A Pire::HalfFinalScanner run over ONE string resident in HBM, counted by the whole GPU (pire_gpu_count_string):
    ``Result(r)`` is the number of positions where a match of regexp r ends.  ``Run(text)`` may be called many times:
    the texts are counted as one string, the state carried from call to call in a device word and the counts added to
    a zeroed device tensor of u64 (``Counts()``), so chained calls do not synchronise.  ``state`` = a StateIndex to
    resume from (not counted again: the run that reached it counted it), None = Initialize() (counted).  Every
    ``Run()`` launches at once on the current stream; ``Begin()`` is folded into the first launch, ``End()`` is a launch
    of its own.  Results (``Result()``, ``AcceptedRegexps()``, ``Final()``, ``State()``) synchronise."""

    def __init__(self, sc, state=None):
        self.Sc = sc
        self._start = None if state is None else int(state)
        self._words = None         # device: [StateIndex, match word]
        self._counts = None        # device: max(1, regexps) u64
        self._begin = False
        self._ran = False

    def Begin(self):
        if self._ran:
            raise ValueError("Begin() must precede Run()")
        self._begin = True
        return self

    def Run(self, text):
        torch = _torch()
        if text.dtype != torch.uint8 or not text.is_cuda or not text.is_contiguous() or text.device.index != self.Sc.device:
            raise ValueError("text must be a contiguous uint8 CUDA tensor on the scanner's device")
        self._launch(text, 0)
        return self

    def End(self):
        self._launch(None, N.RUN_END)
        return self

    def _launch(self, text, flags):
        if self._begin:
            flags |= N.RUN_BEGIN
            self._begin = False
        start = stream = words = counts = None
        if self.Sc.device >= 0:
            torch = _torch()
            dev = torch.device("cuda", self.Sc.device)
            if self._words is None:
                self._words = torch.empty(2, dtype=torch.int32, device=dev)
                self._counts = torch.zeros(max(1, self.Sc.RegexpsCount()), dtype=torch.int64, device=dev)
                if self._start is not None:
                    word = self._start & 0xFFFFFFFF
                    self._words[0] = word - (1 << 32) if word >= (1 << 31) else word
            stream = torch.cuda.current_stream(dev).cuda_stream
            if self._ran or self._start is not None:
                start = self._words.data_ptr()
            words, counts = self._words.data_ptr(), self._counts.data_ptr()
        N.check(N.lib.pire_gpu_count_string(self.Sc._h, None if text is None else text.data_ptr(), 0 if text is None else text.numel(),
                                            flags, start, counts, None if words is None else words + 4, words, stream),
                "pire_gpu_count_string")
        self._ran = True

    def _results(self):
        if not self._ran:
            self._launch(None, 0)          # nothing run yet: the start state itself (after Begin() if it was asked for)
        return self._words.cpu().numpy().view(np.uint32)

    def Counts(self):
        """The device tensor of counters (int64 holding u64), one per regexp; does not synchronise."""
        if not self._ran:
            self._launch(None, 0)
        return self._counts

    def Result(self, regexp_id):
        """State::Result(regexp_id) (half_final.h:88-90)."""
        return int(self.Counts()[regexp_id].item())

    def AcceptedRegexps(self):
        """HalfFinalScanner::AcceptedRegexps (half_final.h:130-133): regexps with a non-zero counter."""
        return [int(r) for r in np.nonzero(self.Counts().cpu().numpy())[0]]

    def State(self):
        """StateIndex() of the state reached (reference numbering); 0xFFFFFFFF for a start outside the scanner."""
        return int(self._results()[0])

    def Final(self):
        return bool(self._results()[1] & 1)


class StringMatchEnds:
    """Where the matches ``StringCounter`` counts end (pire_gpu_match_ends_string): one entry (end, regexp id) for every
    count, in walk order, where end is the number of bytes consumed (over all ``Run()`` calls) when the final state was
    entered.  The entries go to device tensors of ``capacity`` entries; ``FoundTensor()`` counts all of them, even past
    the capacity, whose entries are dropped (the written ones are then the answer's first ``capacity``).  ``Run(text)``
    may be called many times with no synchronise: the state is carried in a device word and the running byte offset on
    the host.  ``state`` = a StateIndex to resume from (not reported again), None = Initialize() (reported).
    ``Begin()`` is folded into the first launch, ``End()`` is a launch of its own.  ``EndsTensor()``, ``IdsTensor()`` and
    ``FoundTensor()`` do not synchronise; ``Found()``, ``Ends()``, ``Ids()``, ``Final()`` and ``State()`` do."""

    def __init__(self, sc, capacity, state=None):
        self.Sc = sc
        self.capacity = int(capacity)
        self._start = None if state is None else int(state)
        self._words = None         # device: [StateIndex, match word]
        self._ends = self._ids = self._found = None
        self._base = 0             # bytes run so far
        self._begin = False
        self._ran = False

    def Begin(self):
        if self._ran:
            raise ValueError("Begin() must precede Run()")
        self._begin = True
        return self

    def Run(self, text):
        torch = _torch()
        if text.dtype != torch.uint8 or not text.is_cuda or not text.is_contiguous() or text.device.index != self.Sc.device:
            raise ValueError("text must be a contiguous uint8 CUDA tensor on the scanner's device")
        self._launch(text, 0)
        return self

    def End(self):
        self._launch(None, N.RUN_END)
        return self

    def _launch(self, text, flags):
        if self._begin:
            flags |= N.RUN_BEGIN
            self._begin = False
        start = stream = words = ends = ids = found = None
        if self.Sc.device >= 0:
            torch = _torch()
            dev = torch.device("cuda", self.Sc.device)
            if self._words is None:
                self._words = torch.empty(2, dtype=torch.int32, device=dev)
                self._ends = torch.empty(self.capacity, dtype=torch.int64, device=dev)
                self._ids = torch.empty(self.capacity, dtype=torch.int32, device=dev)
                self._found = torch.zeros(1, dtype=torch.int64, device=dev)
                if self._start is not None:
                    word = self._start & 0xFFFFFFFF
                    self._words[0] = word - (1 << 32) if word >= (1 << 31) else word
            stream = torch.cuda.current_stream(dev).cuda_stream
            if self._ran or self._start is not None:
                start = self._words.data_ptr()
            words, ends, ids, found = self._words.data_ptr(), self._ends.data_ptr(), self._ids.data_ptr(), self._found.data_ptr()
        n = 0 if text is None else text.numel()
        N.check(N.lib.pire_gpu_match_ends_string(self.Sc._h, None if text is None else text.data_ptr(), n, flags, start, self._base,
                                                 ends, ids, self.capacity, found, None if words is None else words + 4, words,
                                                 stream), "pire_gpu_match_ends_string")
        self._base += n
        self._ran = True

    def _ready(self):
        if not self._ran:
            self._launch(None, 0)          # nothing run yet: the start state itself (after Begin() if it was asked for)

    def EndsTensor(self):
        """The device tensor of ends (int64 holding u64), ``capacity`` long; does not synchronise."""
        self._ready()
        return self._ends

    def IdsTensor(self):
        """The device tensor of regexp ids (int32 holding u32), ``capacity`` long; does not synchronise."""
        self._ready()
        return self._ids

    def FoundTensor(self):
        """The device word (int64 holding u64) counting every entry, also those past the capacity; does not synchronise."""
        self._ready()
        return self._found

    def Found(self):
        """The number of entries, also those past the capacity."""
        return int(self.FoundTensor().item())

    def Ends(self):
        """The first min(Found(), capacity) ends, as numpy u64."""
        k = min(self.Found(), self.capacity)
        return self._ends[:k].cpu().numpy().view(np.uint64)

    def Ids(self):
        """The first min(Found(), capacity) regexp ids, as numpy u32."""
        k = min(self.Found(), self.capacity)
        return self._ids[:k].cpu().numpy().view(np.uint32)

    def State(self):
        """StateIndex() of the state reached (reference numbering); 0xFFFFFFFF for a start outside the scanner."""
        self._ready()
        return int(self._words.cpu().numpy().view(np.uint32)[0])

    def Final(self):
        self._ready()
        return bool(self._words.cpu().numpy().view(np.uint32)[1] & 1)


class BatchCounter:
    """``StringCounter`` for n streams at once (pire_gpu_count_batch_from): stream i's Pire::HalfFinalScanner state is
    carried in a device tensor of n states and its counts added to row i of an (n, max(1, regexps)) device tensor of u64,
    so a batch of streams arriving in pieces is counted round after round with no synchronise.  Every ``Run(batch)``
    launches at once on the current stream; string i of the batch is the next piece of stream i.  ``states`` (an int32
    CUDA tensor of n StateIndex values) resumes stream i from states[i] (not counted again: the run that reached it
    counted it), None = Initialize() (counted).  ``Begin()`` is folded into the next launch, ``End()`` is a launch of its
    own over n empty strings.  ``Counts()`` and ``StateTensor()`` do not synchronise; ``Result()``, ``AcceptedRegexps()``,
    ``Final()``, ``Matches()`` and ``States()`` do."""

    def __init__(self, sc, n, states=None):
        torch = _torch()
        self.Sc = sc
        self.n = int(n)
        dev = torch.device("cuda", sc.device)
        if states is not None and (states.dtype != torch.int32 or not states.is_cuda or not states.is_contiguous()
                                   or states.device != dev or states.numel() < self.n):
            raise ValueError("states must be a contiguous int32 CUDA tensor of n states on the scanner's device")
        self._start = states
        self._states = torch.empty(self.n, dtype=torch.int32, device=dev)
        self._bits = torch.empty((self.n + 31) // 32, dtype=torch.int32, device=dev)
        self._counts = torch.zeros((self.n, max(1, sc.RegexpsCount())), dtype=torch.int64, device=dev)
        self._begin = False
        self._ran = False          # a launch has written the states

    def Begin(self):
        if self._ran:
            raise ValueError("Begin() must precede Run()")
        self._begin = True
        return self

    def Run(self, batch):
        if batch.trim:
            raise ValueError("line batches have no per-string starts")
        if batch.order is not None:
            raise ValueError("BatchCounter takes no length-ordered batch")
        if batch.n != self.n:
            raise ValueError("BatchCounter.Run needs a batch of n = %d strings, got %d" % (self.n, batch.n))
        if batch.device != self._states.device:
            raise ValueError("the batch must be on the scanner's device")
        self._launch(batch.corpus.data_ptr(), None if batch.offsets is None else batch.offsets.data_ptr(), batch.fixed_len, 0)
        return self

    def End(self):
        self._launch(None, None, 0, N.RUN_END)
        return self

    def _launch(self, corpus, offsets, fixed_len, flags):
        if self._begin:
            flags |= N.RUN_BEGIN
            self._begin = False
        torch = _torch()
        if self._ran:
            start = self._states.data_ptr()
        else:
            start = None if self._start is None else self._start.data_ptr()
        stream = torch.cuda.current_stream(self._states.device).cuda_stream
        N.check(N.lib.pire_gpu_count_batch_from(self.Sc._h, corpus, offsets, fixed_len, self.n, flags, start,
                                                self._counts.data_ptr(), self._bits.data_ptr(), self._states.data_ptr(),
                                                stream), "pire_gpu_count_batch_from")
        self._ran = True

    def _ensure(self):
        if not self._ran:
            self._launch(None, None, 0, 0)      # nothing run yet: the start states (after Begin() if it was asked for)

    # without a synchronise ------------------------------------------------------------
    def Counts(self):
        """The device tensor (n, max(1, regexps)) of counters (int64 holding u64); row i is stream i's."""
        self._ensure()
        return self._counts

    def StateTensor(self):
        """The device tensor (int32, n) of the states reached, reference numbering: the ``states`` of a later
        BatchCounter."""
        self._ensure()
        return self._states

    # synchronising --------------------------------------------------------------------
    def Result(self, i, regexp_id):
        """State::Result(regexp_id) of stream i (half_final.h:88-90)."""
        return int(self.Counts()[i, regexp_id].item())

    def AcceptedRegexps(self, i):
        """HalfFinalScanner::AcceptedRegexps (half_final.h:130-133) of stream i: regexps with a non-zero counter."""
        return [int(r) for r in np.nonzero(self.Counts()[i].cpu().numpy())[0]]

    def Matches(self):
        """numpy bool[n]: Final() of each stream's state."""
        self._ensure()
        words = self._bits.cpu().numpy().view(np.uint32)
        return np.unpackbits(words.view(np.uint8), bitorder="little")[: self.n].astype(bool)

    def Final(self, i):
        return bool(self.Matches()[i])

    def States(self):
        """StateIndex() of each stream's state (reference numbering); 0xFFFFFFFF for a start outside the scanner."""
        return self.StateTensor().cpu().numpy().view(np.uint32)


class BatchMatchEnds:
    """Where the matches ``BatchCounter`` counts end (pire_gpu_match_ends_batch_from): one entry (stream, end, regexp id)
    for every count, ordered by stream, then in walk order within a stream, where end is the number of bytes of that
    stream consumed (over all ``Run()`` calls) when the final state was entered.  The entries go to device tensors of
    ``capacity`` entries; ``FoundTensor()`` counts all of them, even past the capacity, whose entries are dropped (the
    written ones are then the answer's first ``capacity``).  Every ``Run(batch)`` launches at once on the current stream,
    string i of the batch being the next piece of stream i, and appends its entries; the states and the streams' byte
    offsets are carried in device tensors, so rounds need no synchronise.  ``states`` (an int32 CUDA tensor of n
    StateIndex values) resumes stream i from states[i] (not reported again), None = Initialize() (reported).
    ``Begin()`` is folded into the next launch, ``End()`` is a launch of its own over n empty strings.
    ``StringsTensor()``, ``EndsTensor()``, ``IdsTensor()``, ``FoundTensor()``, ``StateTensor()`` and ``PosTensor()`` do
    not synchronise; ``Found()``, ``Strings()``, ``Ends()``, ``Ids()``, ``Matches()`` and ``States()`` do."""

    def __init__(self, sc, n, capacity, states=None):
        torch = _torch()
        self.Sc = sc
        self.n = int(n)
        self.capacity = int(capacity)
        dev = torch.device("cuda", sc.device)
        if states is not None and (states.dtype != torch.int32 or not states.is_cuda or not states.is_contiguous()
                                   or states.device != dev or states.numel() < self.n):
            raise ValueError("states must be a contiguous int32 CUDA tensor of n states on the scanner's device")
        self._start = states
        self._states = torch.empty(self.n, dtype=torch.int32, device=dev)
        self._bits = torch.empty((self.n + 31) // 32, dtype=torch.int32, device=dev)
        self._pos = torch.zeros(self.n, dtype=torch.int64, device=dev)
        self._strings = torch.empty(self.capacity, dtype=torch.int32, device=dev)
        self._ends = torch.empty(self.capacity, dtype=torch.int64, device=dev)
        self._ids = torch.empty(self.capacity, dtype=torch.int32, device=dev)
        self._found = torch.zeros(1, dtype=torch.int64, device=dev)
        self._begin = False
        self._ran = False          # a launch has written the states

    def Begin(self):
        if self._ran:
            raise ValueError("Begin() must precede Run()")
        self._begin = True
        return self

    def Run(self, batch):
        if batch.trim:
            raise ValueError("line batches have no per-string starts")
        if batch.order is not None:
            raise ValueError("BatchMatchEnds takes no length-ordered batch")
        if batch.n != self.n:
            raise ValueError("BatchMatchEnds.Run needs a batch of n = %d strings, got %d" % (self.n, batch.n))
        if batch.device != self._states.device:
            raise ValueError("the batch must be on the scanner's device")
        self._launch(batch.corpus.data_ptr(), None if batch.offsets is None else batch.offsets.data_ptr(), batch.fixed_len, 0)
        return self

    def End(self):
        self._launch(None, None, 0, N.RUN_END)
        return self

    def _launch(self, corpus, offsets, fixed_len, flags):
        if self._begin:
            flags |= N.RUN_BEGIN
            self._begin = False
        torch = _torch()
        if self._ran:
            start = self._states.data_ptr()
        else:
            start = None if self._start is None else self._start.data_ptr()
        stream = torch.cuda.current_stream(self._states.device).cuda_stream
        N.check(N.lib.pire_gpu_match_ends_batch_from(self.Sc._h, corpus, offsets, fixed_len, self.n, flags, start,
                                                     self._pos.data_ptr(), self._strings.data_ptr(), self._ends.data_ptr(),
                                                     self._ids.data_ptr(), self.capacity, self._found.data_ptr(),
                                                     self._bits.data_ptr(), self._states.data_ptr(), stream),
                "pire_gpu_match_ends_batch_from")
        self._ran = True

    def _ensure(self):
        if not self._ran:
            self._launch(None, None, 0, 0)      # nothing run yet: the start states (after Begin() if it was asked for)

    # without a synchronise ------------------------------------------------------------
    def StringsTensor(self):
        """The device tensor of stream indices (int32 holding u32), ``capacity`` long."""
        self._ensure()
        return self._strings

    def EndsTensor(self):
        """The device tensor of ends (int64 holding u64), ``capacity`` long."""
        self._ensure()
        return self._ends

    def IdsTensor(self):
        """The device tensor of regexp ids (int32 holding u32), ``capacity`` long."""
        self._ensure()
        return self._ids

    def FoundTensor(self):
        """The device word (int64 holding u64) counting every entry, also those past the capacity."""
        self._ensure()
        return self._found

    def StateTensor(self):
        """The device tensor (int32, n) of the states reached, reference numbering: the ``states`` of a later
        BatchCounter or BatchMatchEnds."""
        self._ensure()
        return self._states

    def PosTensor(self):
        """The device tensor (int64 holding u64, n) of the bytes each stream has consumed so far."""
        self._ensure()
        return self._pos

    # synchronising --------------------------------------------------------------------
    def Found(self):
        """The number of entries, also those past the capacity."""
        return int(self.FoundTensor().item())

    def Strings(self):
        """The first min(Found(), capacity) stream indices, as numpy u32."""
        k = min(self.Found(), self.capacity)
        return self._strings[:k].cpu().numpy().view(np.uint32)

    def Ends(self):
        """The first min(Found(), capacity) ends, as numpy u64."""
        k = min(self.Found(), self.capacity)
        return self._ends[:k].cpu().numpy().view(np.uint64)

    def Ids(self):
        """The first min(Found(), capacity) regexp ids, as numpy u32."""
        k = min(self.Found(), self.capacity)
        return self._ids[:k].cpu().numpy().view(np.uint32)

    def Matches(self):
        """numpy bool[n]: Final() of each stream's state."""
        self._ensure()
        words = self._bits.cpu().numpy().view(np.uint32)
        return np.unpackbits(words.view(np.uint8), bitorder="little")[: self.n].astype(bool)

    def States(self):
        """StateIndex() of each stream's state (reference numbering); 0xFFFFFFFF for a start outside the scanner."""
        return self.StateTensor().cpu().numpy().view(np.uint32)


NO_START = 0xFFFFFFFFFFFFFFFF


class MatchStartsResult:
    """What ``MatchStarts`` wrote: per match-ends entry, the leftmost start of its match and whether that start could
    move further left with more bytes on the left of the window.  ``StartsTensor()`` and ``OpenTensor()`` do not
    synchronise; ``Starts()`` and ``Open()`` do."""

    def __init__(self, ends, starts, open_):
        self._ends, self._starts, self._open = ends, starts, open_

    def StartsTensor(self):
        """The device tensor of starts (int64 holding u64, NO_START = none), the ends' ``capacity`` long; entries whose
        end lies outside the window keep NO_START."""
        return self._starts

    def OpenTensor(self):
        """The device tensor (uint8) of open flags, the ends' ``capacity`` long."""
        return self._open

    def Starts(self):
        """The first min(Found(), capacity) starts, as numpy u64."""
        k = min(self._ends.Found(), self._ends.capacity)
        return self._starts[:k].cpu().numpy().view(np.uint64)

    def Open(self):
        """The first min(Found(), capacity) open flags, as numpy bool."""
        k = min(self._ends.Found(), self._ends.capacity)
        return self._open[:k].cpu().numpy().astype(bool)


def MatchStarts(rsc, ends, window, base=0, begin=True, end=True, max_back=0):
    """Where the matches ``ends`` lists start (pire_gpu_match_starts_string / _batch): Pire::LongestSuffix through
    ``rsc``, a Scanner of the same patterns built with Fsm::Reverse() (glued in the same order), walked leftwards from
    each entry's end and testing the entry's regexp id.  ``ends`` is a ``StringMatchEnds`` whose window is a uint8 CUDA
    tensor holding the text bytes at positions [base, base + numel), or a ``BatchMatchEnds`` whose window is the
    ``Batch`` of its last round (each stream's window ends where ``PosTensor()`` says).  ``begin`` says that the window
    starts where the text begins (BeginMark), ``end`` that the text ended with End() (EndMark); ``max_back`` > 0 bounds
    every walk.  Entries outside the window are left as NO_START.  Launches on the current stream, no synchronise."""
    torch = _torch()
    flags = (N.RUN_BEGIN if begin else 0) | (N.RUN_END if end else 0)
    if not isinstance(ends, (StringMatchEnds, BatchMatchEnds)):
        raise TypeError("ends must be a StringMatchEnds or a BatchMatchEnds")
    dev = ends.EndsTensor().device
    starts = torch.full((ends.capacity,), -1, dtype=torch.int64, device=dev)
    open_ = torch.zeros(ends.capacity, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    if ends.capacity == 0:
        pass                                              # no entries to walk (and no buffers to pass)
    elif isinstance(ends, StringMatchEnds):
        if window.dtype != torch.uint8 or not window.is_cuda or not window.is_contiguous() or window.device != dev:
            raise ValueError("window must be a contiguous uint8 CUDA tensor on the scanner's device")
        N.check(N.lib.pire_gpu_match_starts_string(rsc._h, window.data_ptr(), window.numel(), int(base), flags, int(max_back),
                                                   ends.EndsTensor().data_ptr(), ends.IdsTensor().data_ptr(), None,
                                                   ends.FoundTensor().data_ptr(), ends.capacity, starts.data_ptr(),
                                                   open_.data_ptr(), stream), "pire_gpu_match_starts_string")
    else:
        if window.trim or window.order is not None or window.n != ends.n or window.device != dev:
            raise ValueError("window must be a plain batch of the ends' n streams on the scanner's device")
        N.check(N.lib.pire_gpu_match_starts_batch(rsc._h, window.corpus.data_ptr(),
                                                  None if window.offsets is None else window.offsets.data_ptr(),
                                                  window.fixed_len, window.n, ends.PosTensor().data_ptr(), flags,
                                                  int(max_back), ends.StringsTensor().data_ptr(), ends.EndsTensor().data_ptr(),
                                                  ends.IdsTensor().data_ptr(), None, ends.FoundTensor().data_ptr(),
                                                  ends.capacity, starts.data_ptr(), open_.data_ptr(), stream),
                "pire_gpu_match_starts_batch")
    return MatchStartsResult(ends, starts, open_)


def Runner(sc, states=None):
    """Pire::Runner(sc) (run.h:388-389); with ``states`` Pire::Runner(sc, st) (run.h:391-392) for every string."""
    return RunHelper(sc, states)


def Matches(sc, batch):
    """Pire::Matches(scanner, begin, end) (run.h:396-400): Run without Begin/End marks."""
    return Runner(sc).Run(batch).Matches()


def _prefix(sc, batch, shortest, throughBeginMark, throughEndMark, suffix=False):
    torch = _torch()
    out = torch.empty(batch.n, dtype=torch.int32, device=batch.device)
    flags = (N.RUN_BEGIN if throughBeginMark else 0) | (N.RUN_END if throughEndMark else 0) | (N.RUN_LINES if batch.trim else 0)
    stream = torch.cuda.current_stream(batch.device).cuda_stream
    fn = N.lib.pire_gpu_suffix_batch if suffix else N.lib.pire_gpu_prefix_batch
    N.check(fn(sc._h, batch.corpus.data_ptr(), batch.offsets.data_ptr() if batch.offsets is not None else None,
               batch.fixed_len, batch.n, flags, int(shortest), out.data_ptr(), stream),
            "pire_gpu_suffix_batch" if suffix else "pire_gpu_prefix_batch")
    res = out.cpu().numpy().view(np.uint32).astype(np.int64)
    res[res == 0xFFFFFFFF] = -1
    return res


def LongestPrefix(sc, batch, throughBeginMark=False, throughEndMark=False):
    """Pire::LongestPrefix (run.h:277-292) per string: prefix length, or -1 where the reference returns null."""
    return _prefix(sc, batch, False, throughBeginMark, throughEndMark)


def ShortestPrefix(sc, batch, throughBeginMark=False, throughEndMark=False):
    """Pire::ShortestPrefix (run.h:294-311) per string: prefix length, or -1 where the reference returns null."""
    return _prefix(sc, batch, True, throughBeginMark, throughEndMark)


def LongestSuffix(sc, batch, throughEndMark=False, throughBeginMark=False):
    """Pire::LongestSuffix (run.h:316-342) per string, walked from its last byte: suffix length, or -1 for null."""
    return _prefix(sc, batch, False, throughBeginMark, throughEndMark, suffix=True)


def ShortestSuffix(sc, batch, throughEndMark=False, throughBeginMark=False):
    """Pire::ShortestSuffix (run.h:345-362) per string: suffix length, or -1 for null."""
    return _prefix(sc, batch, True, throughBeginMark, throughEndMark, suffix=True)


class HalfFinalResult:
    """What a batch of HalfFinalScanner states reports (half_final.h:58-120)."""

    def __init__(self, counts, final):
        self.counts, self.final = counts, final

    def Result(self, i, regexp_id):
        """State::Result(regexp_id) of string i (half_final.h:88-90)."""
        return int(self.counts[i, regexp_id])

    def AcceptedRegexps(self, i):
        """HalfFinalScanner::AcceptedRegexps (half_final.h:130-133): regexps with a non-zero counter."""
        return [int(r) for r in np.nonzero(self.counts[i])[0]]

    def Final(self, i):
        return bool(self.final[i])


def HalfFinalCount(sc, batch, begin=True, end=True):
    """Per string: Initialize; [Step(BeginMark)]; Run; [Step(EndMark)] of a Pire::HalfFinalScanner
    (half_final.h:136-163, driven as tests/count_ut.cpp:54-63 does) -> HalfFinalResult with
    counts[n, regexps] (numpy u32) and final[n] (bool).  `sc` is a Scanner loaded from the
    HalfFinalScanner's Save() stream."""
    torch = _torch()
    regs = max(1, sc.RegexpsCount())
    counts = torch.empty((batch.n, regs), dtype=torch.int32, device=batch.device)
    bits = torch.zeros((batch.n + 31) // 32, dtype=torch.int32, device=batch.device)
    flags = (N.RUN_BEGIN if begin else 0) | (N.RUN_END if end else 0) | (N.RUN_LINES if batch.trim else 0)
    stream = torch.cuda.current_stream(batch.device).cuda_stream
    N.check(N.lib.pire_gpu_count_batch(sc._h, batch.corpus.data_ptr(),
                                       batch.offsets.data_ptr() if batch.offsets is not None else None,
                                       batch.fixed_len, batch.n, flags, counts.data_ptr(), bits.data_ptr(), stream),
            "pire_gpu_count_batch")
    words = bits.cpu().numpy().view(np.uint32)
    final = ((words[np.arange(batch.n) // 32] >> (np.arange(batch.n) % 32).astype(np.uint32)) & 1).astype(bool)
    return HalfFinalResult(counts.cpu().numpy().view(np.uint32), final)
