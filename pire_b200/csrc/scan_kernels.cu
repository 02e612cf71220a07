// scan_kernels.cu -- hand-written sm_90a kernels for Pire's inner scan loop.
//
// Replaces, for a batch of strings, the reference's
//     Runner(sc).Begin().Run(ptr,len).End()   (pire/run.h:365-392)
// whose per-byte body is  state = row(state)[letter_of[byte]]
// (Step run.h:50-57 -> Next/Translate/NextTranslated multi.h:163-192), including
// the ExitMasks early return on NoExit states (multi.h:955-958).
//
// Mapping to the machine (one input string per warp lane):
//   * The table of hot rows (dfa_tables.hpp) is staged once per persistent CTA
//     into shared memory with a 1-D TMA bulk copy (cp.async.bulk + mbarrier).
//   * A lane keeps its state as a hot id g in 0..H (H = "not in the table").
//     One step is   bb = IDP.4A(word, 1 << 8k, base)  (input byte k plus the table's
//     256-byte aligned shared address, FMA pipe; PRMT in the prefix kernels; independent
//     of g, so it runs ahead),
//     addr = IMAD(g, 292, bb)  (rows are 292 bytes apart: consecutive rows start nine
//     banks apart, which spreads the conflicts between lanes in different rows),
//     g = LDS.U8 [addr].  No class lookup, no branch.
//   * kPred variant: the LDS is predicated off while the lane sits in hot id 0
//     and the byte cannot leave it (32-slot bitmap probed with a funnel shift),
//     so fewer lanes hit the banks and the load costs fewer wavefronts.
//   * LOOK variant (the glued benchmark scan): the filter looks one byte further -- a resting
//     lane reads the table only if this byte and the next both pass -- in 5.5 instructions per
//     byte (LookProbe / LookStep), two strings per lane (ScanUniformLookRingKernel, fed from a per-lane cp.async ring
//     with two blocks of each string in flight).  The LOOK_RING1 variant walks
//     one string per lane from such a ring, 32 warps per SM (ScanUniformLookRing1Kernel).
//   * Input bytes: each lane streams its own string: 32-byte read-only loads (two
//     LDG.128 of one sector, the second an L1 hit), one ahead in a register ping-pong (uniform kernels,
//     two LDG.128 per 32 bytes), or a four-deep cp.async ring of 16-byte chunks in shared memory
//     (CSR kernels).  Long strings of a length-ordered batch are split over a warp
//     (ScanSplitKernel), one string given alone over the whole grid (ScanStringKernel); lines of text are scanned
//     in stream (ScanTextKernel).
//   * Prefix / suffix scans and HalfFinalScanner counting reuse the walk; final hot
//     states carry the highest ids, so a running maximum per chunk says whether any
//     step needs the per-byte work.
//   * A lane whose walk leaves the hot rows reads H from then on (row H is a
//     sink); after the chunk the lane is replayed byte by byte through the
//     complete class-indirect table in global memory / L2.
//   * End(): one 8-byte load of the precomputed per-state report; the match bit
//     of 32 strings is assembled with a warp ballot and written as one word.
// There is no dense contraction anywhere on this path, hence no tensor cores.

#include "scan_kernels.cuh"

#include <atomic>
#include <mutex>
#include <cstdlib>
#include <type_traits>

#include <cooperative_groups.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

// One dynamic shared-memory array for every kernel of this file.  The hot rows sit at its start (behind
// the lane-private region in the PRIV kernel, a multiple of 16 KB), 256-byte aligned: FastStep ORs the input
// byte into the table's shared-window address with one PRMT.  The array is declared with 1 KiB alignment so
// that the alignment is a property of the build; StageTables keeps a trap as a backstop.
extern "C" {
extern __shared__ __align__(1024) uint8_t pire_b200_smem[];
}

namespace pire_b200 {

namespace {

constexpr int kBlock = 512;
constexpr int kMinBlocksPerSM = 3;
// The generic kernel keeps 64 + 64 bytes of input per lane in registers and runs at two
// CTAs per SM: ragged batches are bound by the latency of their longest strings (one
// dependent LDS chain per string), which fewer co-resident warps shorten.
constexpr int kGenericBlocksPerSM = 2;
constexpr int kWarpsPerBlock = kBlock / 32;
// Grid cap of the grid-stride helper kernels (line counting, synthesis, accept gathering): `per_sm` CTAs on every SM
// of the current device.
unsigned long long GridCap(unsigned per_sm)
{
    int device = 0, sms = 0;
    if (cudaGetDevice(&device) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms < 1)
        sms = 1;
    return (unsigned long long) sms * per_sm;
}

std::atomic<uint64_t> g_launches{0};

// ---------------------------------------------------------------- PTX helpers

__device__ __forceinline__ uint32_t SmemAddr(const void* p)
{
    return (uint32_t) __cvta_generic_to_shared(p);
}

__device__ __forceinline__ void MbarInit(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(SmemAddr(bar)), "r"(count) : "memory");
}

__device__ __forceinline__ void FenceBarrierInit()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void MbarExpectTx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(SmemAddr(bar)), "r"(bytes) : "memory");
}

__device__ __forceinline__ void MbarWait(uint64_t* bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(SmemAddr(bar)), "r"(parity) : "memory");
}

// 1-D TMA bulk copy global -> shared, completion signalled on an mbarrier.
__device__ __forceinline__ void BulkCopyG2S(void* dst, const void* src, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(SmemAddr(dst)),
                 "l"(src), "r"(bytes), "r"(SmemAddr(bar))
                 : "memory");
}

// Asynchronous 16-byte copy global -> shared (LDGSTS).  Completion is tracked by
// commit/wait groups, not by the register scoreboard, so a pending copy never makes an
// unrelated shared-memory load wait for DRAM (which is what register prefetch did in the
// generic kernel: one exposed DRAM round trip per iteration, r01 experiments).
__device__ __forceinline__ void CopyAsync16(uint32_t dst_shared, const uint8_t* src)
{
    asm volatile("cp.async.cg.shared.global.L2::256B [%0], [%1], 16;" ::"r"(dst_shared), "l"(src) : "memory");
}
__device__ __forceinline__ void CopyAsyncCommit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void CopyAsyncWait() { asm volatile("cp.async.wait_group %0;" ::"n"(kPending) : "memory"); }

__device__ __forceinline__ uint4 LoadShared16(uint32_t shared_addr)
{
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(shared_addr) : "memory");
    return v;
}

// Streaming read-only load of the corpus (uniform kernels): 32 bytes = one full sector per
// lane per request, never re-used by this SM.
// L2 prefetch of the 128-byte line at p: no destination registers, so nothing tempts the scheduler to delay it.
__device__ __forceinline__ void PrefetchL2(const uint8_t* p)
{
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

// The same load with a 256-byte L2 prefetch: the first touch of a 256-byte region of a string brings all of it
// into L2, so the following seven 32-byte loads of the lane are L2 hits.  sm_90 has no 256-bit load: the 32 bytes
// are two 128-bit loads of the same sector, issued back to back.  Both allocate in L1, so the second half of the
// sector is an L1 hit; with L1::no_allocate both halves went to L2, and on an H100 the scans ran at about 0.55 of
// the speed (glued scan 769 against 1393 GB/s, same build otherwise).
__device__ __forceinline__ void LoadStream32P(const uint8_t* p, uint4& a, uint4& b)
{
    asm volatile("ld.global.nc.L2::256B.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
                 "ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                 : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w), "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w)
                 : "l"(p));
}

// The uniform kernels' load: the first half carries the 128-byte L2 prefetch-size hint, so an L2 miss fetches the
// sector's whole 128-byte line and HBM serves whole lines instead of scattered 32-byte sectors (the three other
// sectors of the line are the lane's next three blocks).  The lines of every string in progress stay in L2: at most
// 132 SMs x 48 warps x 32 strings x 128 B = 26 MB on an H100, of its 50 MB.  The 256-byte hint would take twice that,
// and the two-strings-per-lane kernel (29 MB at 128 B) measured slower with it.
__device__ __forceinline__ void LoadStream32(const uint8_t* p, uint4& a, uint4& b)
{
    asm volatile("ld.global.nc.L2::128B.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
                 "ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                 : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w), "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w)
                 : "l"(p));
}

// ---------------------------------------------------------------- shared layout

constexpr int kStageSlots = 4;                                      // 16-byte chunks in flight per lane
constexpr size_t kStageBytes = (size_t) 512 * kStageSlots * 16;      // generic kernel: 32 KB per CTA

struct SharedView {
    uint8_t* priv;       // (priv_rows/4) * 16 KB, PRIV variant only (else empty)
    uint8_t* hot;        // (H+1)*256
    uint16_t* cls;       // 256
    uint8_t* noexit;     // 256 (H+1 used)
    uint64_t* bar;
    uint8_t* stage;      // generic kernel only: cp.async ring, kStageBytes
};

__host__ __device__ inline size_t HotBytes(uint32_t hot) { return (size_t) ((hot + 1 + 3) / 4 * 4) * kHotStride; }   // == HotTableBytes

__host__ __device__ inline size_t PrivBytes(uint32_t priv_rows) { return (size_t) (priv_rows / 4) * 16384; }

__device__ __forceinline__ SharedView CarveShared(uint8_t* smem, uint32_t hot, uint32_t priv_rows = 0)
{
    SharedView v;
    v.priv = smem;
    smem += PrivBytes(priv_rows);
    v.hot = smem;
    v.cls = reinterpret_cast<uint16_t*>(smem + HotBytes(hot));
    v.noexit = smem + HotBytes(hot) + 512;
    v.bar = reinterpret_cast<uint64_t*>(smem + HotBytes(hot) + 512 + 256);
    v.stage = smem + HotBytes(hot) + 512 + 256 + 16;
    return v;
}

// Stage the tables: hot rows by TMA bulk copy, the two small tables by plain loads.
__device__ __forceinline__ void StageTables(const ScanArgs& a, const SharedView& sv, const uint8_t* hot8, uint32_t hot)
{
    const uint32_t total = (uint32_t) HotBytes(hot);
    if ((SmemAddr(sv.hot) & 255u) != 0)
        __trap();                          // FastStep builds base | byte with one PRMT
    if (threadIdx.x == 0) {
        MbarInit(sv.bar, 1);
        FenceBarrierInit();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        MbarExpectTx(sv.bar, total);
        constexpr uint32_t kPiece = 16384;
        for (uint32_t off = 0; off < total; off += kPiece) {
            uint32_t n = total - off < kPiece ? total - off : kPiece;
            BulkCopyG2S(sv.hot + off, hot8 + off, n, sv.bar);
        }
    }
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) {
        sv.cls[i] = a.cls[i];
        sv.noexit[i] = i <= hot ? a.noexit[i] : 0;
    }
    MbarWait(sv.bar, 0);
    __syncthreads();
}

// ---------------------------------------------------------------- the walk

struct Tables {
    const uint8_t* hot;
    const uint16_t* cls;
    const void* full;
    uint32_t H;
    uint32_t letters;
    uint32_t wide;
    uint32_t m0;              // 32-slot exit bitmap of hot id 0, slot = byte & 31
    uint32_t base;            // shared-window address of the hot rows; 256-byte aligned (FastStep relies on it)
};

// One byte through the complete table (hot rows first: they are in shared memory).
__device__ __forceinline__ uint32_t SlowStep(const Tables& t, uint32_t s, uint32_t b)
{
    if (s < t.H) {
        uint32_t h = t.hot[s * kHotStride + b];
        if (h != t.H)
            return h;
    }
    size_t at = (size_t) s * t.letters + t.cls[b];
    return t.wide ? __ldg(static_cast<const uint32_t*>(t.full) + at) : (uint32_t) __ldg(static_cast<const uint16_t*>(t.full) + at);
}

// Lane state: g in 0..H; when g == H the real state is `cold`.
struct LaneState {
    uint32_t g;
    uint32_t cold;
};

__device__ __forceinline__ uint32_t FullState(const Tables& t, const LaneState& s) { return s.g == t.H ? s.cold : s.g; }

__device__ __forceinline__ void SetFull(const Tables& t, LaneState& s, uint32_t full)
{
    if (full < t.H) {
        s.g = full;
    } else {
        s.g = t.H;
        s.cold = full;
    }
}

template <bool kPred, bool kIdp = true>
__device__ __forceinline__ void FastStep(const Tables& t, uint32_t& g, uint32_t w, uint32_t sel)
{
    // Entry of (id g, byte b) sits at base + g * kHotStride + b.  `bb` = base | b comes from one PRMT (the
    // base is 256-byte aligned, so its low byte is free) and does not depend on g: the dependent chain of a
    // step is IMAD (FMA pipe) -> LDS, as short as the PRMT -> LDS of an unpadded table.
    // byte `sel` + base: IDP.4A on the FMA pipe (the scan, CSR and counting kernels are short of ALU slots), or PRMT on
    // the ALU pipe for the prefix kernels, whose look-ahead pass keeps the FMA side busy
    const uint32_t bb = kIdp ? __dp4a(w, 1u << (8 * (sel & 3u)), t.base) : __byte_perm(w, t.base, 0x7650u | (sel & 3u));
    if (kPred) {
        // bit (byte & 31) of the 32-slot exit bitmap: may this byte leave hot id 0?
        // Lanes resting in id 0 on a self-looping byte skip the load (fewer bank
        // conflicts).  Spelled in PTX so that it stays SHF, LOP3 -> predicate,
        // IMAD, @p LDS.  (Sharper filters -- a 64-slot bitmap probed with SHF.R.U64, or a
        // slot of (byte >> 2) & 31 -- pass fewer lanes (2.12 / 2.14 vs 2.23 modelled
        // wavefronts) but measured 8 % slower: a fourth ALU-pipe instruction per byte,
        // issued at half rate, becomes the bound; DESIGN.md results log.)
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            ".reg .b32 probe, addr;\n"
            "shf.r.wrap.b32 probe, %2, 0, %1;\n"        // the shift amount is bb & 31 == byte & 31
            "and.b32 probe, probe, 1;\n"
            "or.b32 probe, probe, %0;\n"
            "setp.ne.u32 p, probe, 0;\n"
            "mad.lo.u32 addr, %0, %3, %1;\n"
            "@p ld.shared.u8 %0, [addr];\n"
            "}\n"
            : "+r"(g)
            : "r"(bb), "r"(t.m0), "n"(kHotStride));
    } else {
        const uint32_t addr = g * kHotStride + bb;
        asm("ld.shared.u8 %0, [%1];" : "=r"(g) : "r"(addr));
    }
}

template <bool kPred>
__device__ __forceinline__ void FastWord(const Tables& t, uint32_t& g, uint32_t w)
{
    FastStep<kPred>(t, g, w, 0x5540);
    FastStep<kPred>(t, g, w, 0x5541);
    FastStep<kPred>(t, g, w, 0x5542);
    FastStep<kPred>(t, g, w, 0x5543);
}

// Replay of one 16-byte chunk through the complete table, for a lane that was
// (or fell) outside the hot rows.  Out of line and by value: it is rare, and
// keeping it away from the caller keeps the fast loop free of local memory.
__device__ __noinline__ uint32_t ReplayChunk(const uint8_t* hot, const uint16_t* cls, const void* full, uint32_t H,
                                             uint32_t letters_wide, uint32_t from, uint4 v)
{
    Tables t;
    t.hot = hot;
    t.base = SmemAddr(hot);
    t.cls = cls;
    t.full = full;
    t.H = H;
    t.letters = letters_wide & 0x7fffffffu;
    t.wide = letters_wide >> 31;
    t.m0 = 0;
    uint32_t s = from;
#pragma unroll
    for (int k = 0; k < 4; ++k)
        s = SlowStep(t, s, (v.x >> (8 * k)) & 0xffu);
#pragma unroll
    for (int k = 0; k < 4; ++k)
        s = SlowStep(t, s, (v.y >> (8 * k)) & 0xffu);
#pragma unroll
    for (int k = 0; k < 4; ++k)
        s = SlowStep(t, s, (v.z >> (8 * k)) & 0xffu);
#pragma unroll
    for (int k = 0; k < 4; ++k)
        s = SlowStep(t, s, (v.w >> (8 * k)) & 0xffu);
    return s;
}

// 16 input bytes.
template <bool kPred>
__device__ __forceinline__ void Chunk16(const Tables& t, LaneState& s, uint4 v)
{
    const uint32_t before = s.g;
    uint32_t g = s.g;
    FastWord<kPred>(t, g, v.x);
    FastWord<kPred>(t, g, v.y);
    FastWord<kPred>(t, g, v.z);
    FastWord<kPred>(t, g, v.w);
    s.g = g;
    if (g == t.H) {
        uint32_t from = before == t.H ? s.cold : before;
        uint32_t full = ReplayChunk(t.hot, t.cls, t.full, t.H, t.letters | (t.wide << 31), from, v);
        SetFull(t, s, full);
    }
}

// known = false: the string started from a StateIndex outside the scanner (LaneStart); it reports match 0, mask 0 and
// state 0xFFFFFFFF whatever its walk did, and stays out of the match ballot.
__device__ __forceinline__ void Report(const ScanArgs& a, const Tables& t, const LaneState& s, uint64_t unit, uint64_t i, bool valid,
                                       bool known = true)
{
    DeviceFin f = known ? a.fin[FullState(t, s)] : DeviceFin{0u, 0u};
    unsigned matched = __ballot_sync(0xffffffffu, valid && (f.result >> 31));
    if (a.match_bits && (threadIdx.x & 31) == 0)
        a.match_bits[unit] = matched;
    if (valid) {
        if (a.accept_masks)
            a.accept_masks[i] = f.mask;
        if (a.state_idx)
            a.state_idx[i] = known ? f.result & 0x7fffffffu : 0xFFFFFFFFu;
    }
}

// Ordered (length-binned) launches: lane -> string is a permutation, so the match
// bit goes to its word with an atomic OR (the caller zeroes the bitmap).
__device__ __forceinline__ void ReportScattered(const ScanArgs& a, const Tables& t, const LaneState& s, uint64_t i, bool valid,
                                                bool known = true)
{
    if (!valid)
        return;
    DeviceFin f = known ? a.fin[FullState(t, s)] : DeviceFin{0u, 0u};
    if (a.match_bits && (f.result >> 31))
        atomicOr(&a.match_bits[i >> 5], 1u << (i & 31));
    if (a.accept_masks)
        a.accept_masks[i] = f.mask;
    if (a.state_idx)
        a.state_idx[i] = known ? f.result & 0x7fffffffu : 0xFFFFFFFFu;
}

// ---------------------------------------------------------------- starts given by the caller

// One cell of the complete table (global memory / L2).
__device__ __forceinline__ uint32_t FullCell(const Tables& t, uint32_t s, uint32_t cls)
{
    const size_t at = (size_t) s * t.letters + cls;
    return t.wide ? __ldg(static_cast<const uint32_t*>(t.full) + at) : (uint32_t) __ldg(static_cast<const uint16_t*>(t.full) + at);
}

// The state a run starts from when the caller gives it as a StateIndex `old` (reference numbering, Runner(sc, st),
// run.h:391-392): mapped to the new numbering, with BeginMark stepped through the complete table when a.with_begin.  A
// StateIndex at or above Size() reads no table: `known` is cleared and `start` left as it was (the run goes on from it,
// and its result is never reported).
__device__ __forceinline__ void StartFrom(const ScanArgs& a, const Tables& t, uint32_t old, uint32_t& start, bool& known)
{
    known = old < a.states;
    if (known) {
        start = a.new_of_old[old];
        if (a.with_begin)
            start = FullCell(t, start, a.begin_class);
    }
}

// The start of string i in a batch kernel: a.start, or with kStarts its own (a.starts[i], pire_gpu_run_batch_from).  A lane
// past the batch (in_batch false) reads no start.  a.starts may be a.state_idx: every kernel calls this for string i
// before it reports string i.
template <bool kStarts>
__device__ __forceinline__ uint32_t LaneStart(const ScanArgs& a, const Tables& t, uint64_t i, bool in_batch, bool& known)
{
    uint32_t start = a.start;
    known = true;
    if (kStarts && in_batch)
        StartFrom(a, t, a.starts[i], start, known);
    return start;
}

// ---------------------------------------------------------------- kernels

// Uniform batch: fixed length, length % 32 == 0, corpus 32-byte aligned.  kStarts: every string from its own start (LaneStart).
template <bool kPred, bool kStarts>
__global__ void __launch_bounds__(kBlock, kMinBlocksPerSM) ScanUniformKernel(const __grid_constant__ ScanArgs a)
{
    uint8_t* const smem = pire_b200_smem;
    SharedView sv = CarveShared(smem, a.hot);
    StageTables(a, sv, a.hot8, a.hot);

    Tables t;
    t.hot = sv.hot;
    t.base = SmemAddr(sv.hot);
    t.cls = sv.cls;
    t.full = a.full;
    t.H = a.hot;
    t.letters = a.letters;
    t.wide = a.wide;
    t.m0 = a.exit_bitmap0;

    const uint32_t lane = threadIdx.x & 31;
    const uint64_t units = (a.n + 31) / 32;
    const uint64_t warps = (uint64_t) gridDim.x * kWarpsPerBlock;
    const uint32_t len = (uint32_t) a.fixed_len;

    for (uint64_t unit = (uint64_t) blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5); unit < units; unit += warps) {
        const uint64_t i = unit * 32 + lane;
        const bool valid = i < a.n;
        const uint8_t* p = a.corpus + (valid ? i : a.n - 1) * (uint64_t) len;

        LaneState s;
        bool known;
        SetFull(t, s, LaneStart<kStarts>(a, t, i, valid, known));

        if (len != 0) {
            // Two register sets in ping-pong: the 32 bytes after the ones being walked are
            // always in flight (software prefetch, one pair of LDG.128 per lane per 32 bytes).
            uint4 a0, a1, b0, b1;
            LoadStream32(p, a0, a1);
            for (uint32_t off = 0;;) {
                off += 32;
                const bool more_b = off < len;
                if (more_b)
                    LoadStream32(p + off, b0, b1);
                Chunk16<kPred>(t, s, a0);
                Chunk16<kPred>(t, s, a1);
                // multi.h:955-958,:979-982: once no byte can leave any lane's state, the
                // rest of the strings cannot change the outcome.
                if (!more_b || __all_sync(0xffffffffu, sv.noexit[s.g] != 0))
                    break;
                off += 32;
                const bool more_a = off < len;
                if (more_a)
                    LoadStream32(p + off, a0, a1);
                Chunk16<kPred>(t, s, b0);
                Chunk16<kPred>(t, s, b1);
                if (!more_a || __all_sync(0xffffffffu, sv.noexit[s.g] != 0))
                    break;
            }
        }
        Report(a, t, s, unit, i, valid, known);
    }
}

// ---------------------------------------------------------------- LOOK variant
//
// The reference leaves the table walk while a state cannot be left by the bytes ahead (ExitMasks skip loop,
// multi.h:966-989).  The device analogue looks ONE byte further than the round-1 exit filter: a lane resting in
// hot id 0 reads the table only if this byte AND the next one pass the filter F (dfa_tables.hpp: F holds the
// bytes that leave id 0 and the bytes that keep a state entered from id 0 from falling straight back).  If the
// next byte is outside F the lane is back in id 0 after it whatever this byte does, so both reads are skipped
// and the lane never enters the one-step states at all: on random text the lanes outside id 0 drop from 7.4 to
// 5.1 per warp and the active lanes per load from 19 to 12 (host model tools/model_look.cpp: 2.05 -> 1.72
// shared-memory wavefronts per step with the same 32-slot filter; an exact filter would give 1.26).
// A lane that skipped an exit byte is "virtually" in id 0; its true state differs only until the next byte,
// which is outside F and returns it to id 0 on either path, so replays from the register state stay exact.
// The last byte of a string has no successor: it is filtered by F alone.
//
// One step is six instructions, two of them on the dependent chain:
//     bb  = IDP.4A(word, 1 << 8k, base)     byte k + table base, FMA pipe (PRMT in round 1, ALU pipe)
//     pa  = SHF.R.W(F, bb)                  bit (byte & 31) of the filter in bit 0
//     t   = LOP3(pa, pa_next, 1)            both bytes pass
//     p   = LOP3((t | g) != 0)              ... or the lane is outside id 0            [chain]
//     a   = IMAD(g, 292, bb)                                                          [chain]
//     g   = @p LDS.U8 [a]
// k64 = false: 32-slot filter probed with the low five bits of bb (no extra instruction).
// k64 = true : 64-slot filter (slot = byte & 63) probed with SHF.R.U64, which needs the slot alone in a register:
//              one more IDP per byte on the word masked to six bits per byte (FMA pipe, and one LOP3 per word).
//              Printable text folds 3:1 onto 32 slots but only 3:2 onto 64 (model: 1.72 -> 1.42 wavefronts per step).
struct LookFilter {
    uint32_t lo, hi;
    uint32_t zero;      // a kernel argument that is always 0: the addend that keeps the cleaning multiply an IMAD
    uint32_t rev;       // lo with its bits reversed (clean-bit kernels: probes of the odd bytes)
};

// kClean: the probe's bit is moved to bit 31 with the bits below it cleared by one multiply (IMAD, FMA pipe: pa * 2^31
// keeps bit 0 only), so that "both bytes pass, or the lane is outside id 0" is ONE LOP3 with a predicate result over
// (pa, pa_next, g) instead of two: the step keeps six instructions, but two instead of three of them are on the
// half-rate ALU pipe, which the look-ahead kernel keeps busy.
template <bool k64, int kByte, bool kClean = false>
__device__ __forceinline__ void LookProbe(uint32_t w, uint32_t base, const LookFilter& f, uint32_t& bb, uint32_t& pa)
{
    constexpr uint32_t sel = 1u << (8 * kByte);
    bb = __dp4a(w, sel, base);
    if (kClean && (kByte & 1)) {
        // odd bytes: the bit-reversed filter shifted LEFT puts the probe's bit in bit 31 with other filter bits below it.
        // That is good enough: the step ANDs the probes of two neighbouring bytes, one of them is always an even byte,
        // and an even byte's probe is clean -- so an odd byte costs one SHF, an even byte SHF + IMAD: 5.5 instructions
        // per step on average.
        pa = __funnelshift_l(0u, f.rev, bb);
        return;
    }
    if (k64) {
        const uint32_t slot = __dp4a(w & 0x3F3F3F3Fu, sel, 0u);
        pa = (uint32_t) ((((uint64_t) f.hi << 32) | f.lo) >> slot);
    } else {
        pa = __funnelshift_r(f.lo, f.lo, bb);
    }
    if (kClean)
        asm("mad.lo.u32 %0, %1, 0x80000000, %2;" : "=r"(pa) : "r"(pa), "r"(f.zero));
}

template <bool kClean = false>
__device__ __forceinline__ void LookStep(uint32_t& g, uint32_t bb, uint32_t pa, uint32_t pa_next)
{
    if (kClean) {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            ".reg .b32 t, addr;\n"
            "lop3.b32 t, %1, %2, %0, 0xEA;\n"          // (pa & pa_next) | g
            "setp.ne.u32 p, t, 0;\n"
            "mad.lo.u32 addr, %0, %4, %3;\n"
            "@p ld.shared.u8 %0, [addr];\n"
            "}\n"
            : "+r"(g)
            : "r"(pa), "r"(pa_next), "r"(bb), "n"(kHotStride));
        return;
    }
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        ".reg .b32 t, addr;\n"
        "lop3.b32 t, %1, %2, 1, 0x80;\n"
        "or.b32 t, t, %0;\n"
        "setp.ne.u32 p, t, 0;\n"
        "mad.lo.u32 addr, %0, %4, %3;\n"
        "@p ld.shared.u8 %0, [addr];\n"
        "}\n"
        : "+r"(g)
        : "r"(pa), "r"(pa_next), "r"(bb), "n"(kHotStride));
}

// Four bytes.  (bb0, pa0) belong to byte 0 of `w` and were computed by the previous call; pan is the probe of the
// byte that follows the word.  (Looking ahead from the even bytes only -- half a LOP3 less per byte, 1.91 instead of
// 1.72 wavefronts per step in the host model, tools/model_look.cpp -- is not done: it was slower when tried.)
template <bool k64, bool kClean = false>
__device__ __forceinline__ void LookWord(uint32_t& g, uint32_t w, uint32_t bb0, uint32_t pa0, uint32_t pan, uint32_t base,
                                         const LookFilter& f)
{
    uint32_t bb1, bb2, bb3, pa1, pa2, pa3;
    LookProbe<k64, 1, kClean>(w, base, f, bb1, pa1);
    LookProbe<k64, 2, kClean>(w, base, f, bb2, pa2);
    LookProbe<k64, 3, kClean>(w, base, f, bb3, pa3);
    LookStep<kClean>(g, bb0, pa0, pa1);
    LookStep<kClean>(g, bb1, pa1, pa2);
    LookStep<kClean>(g, bb2, pa2, pa3);
    LookStep<kClean>(g, bb3, pa3, pan);
}

// Shared-window address of the dynamic shared memory array, as a link-time constant (a cvta of a generic pointer
// costs an S2R + LEA wherever the compiler chooses to rematerialise it).
__device__ __forceinline__ uint32_t SmemWindowBase()
{
    uint32_t v;
    asm("mov.u32 %0, pire_b200_smem;" : "=r"(v));
    return v;
}

// Thirty-two bytes (one pair of LDG.128 per lane).  next0 = the word that follows the block (ignored when !more: the last
// byte of a string is filtered alone).  A lane that left the hot rows reads the sink row from then on; one test
// per block finds it and replays both 16-byte chunks through the complete table.
// Lane state in two registers: g (hot id, H = outside the hot rows) and prev = the complete state the lane had when
// the block began (its cold state while g == H, else g itself) -- exactly what a replay starts from.
// The replay of a whole 32-byte block for the LOOK kernels: out of line, and with every table pointer read from the
// kernel's parameter block in here, so that the walk loop around the (rare) call carries no argument set-up.
__device__ __noinline__ uint32_t ReplayBlock32(const ScanArgs* a, uint32_t from, uint4 v0, uint4 v1)
{
    const SharedView sv = CarveShared(pire_b200_smem, a->hot);
    const uint32_t letters_wide = a->letters | (a->wide << 31);
    const uint32_t mid = ReplayChunk(sv.hot, sv.cls, a->full, a->hot, letters_wide, from, v0);
    return ReplayChunk(sv.hot, sv.cls, a->full, a->hot, letters_wide, mid, v1);
}

// `late(g)` fetches the first word of the block that follows, after the walk of the block's first 28 bytes: from registers
// loaded a block ahead (ScanUniformLookKernel) or from the ring in shared memory (ScanUniformLookRing1Kernel).
template <bool k64, bool kClean, typename Late>
__device__ __forceinline__ void LookBlock32(const Tables& t, uint32_t& g, uint32_t& prev, const uint4& v0, const uint4& v1,
                                            bool more, const LookFilter& f, Late late, const ScanArgs* args)
{
    prev = g == t.H ? prev : g;
    uint32_t bb, pa, bn, pn;
    LookProbe<k64, 0, kClean>(v0.x, t.base, f, bb, pa);
    LookProbe<k64, 0, kClean>(v0.y, t.base, f, bn, pn);
    LookWord<k64, kClean>(g, v0.x, bb, pa, pn, t.base, f);
    LookProbe<k64, 0, kClean>(v0.z, t.base, f, bb, pa);
    LookWord<k64, kClean>(g, v0.y, bn, pn, pa, t.base, f);
    LookProbe<k64, 0, kClean>(v0.w, t.base, f, bn, pn);
    LookWord<k64, kClean>(g, v0.z, bb, pa, pn, t.base, f);
    LookProbe<k64, 0, kClean>(v1.x, t.base, f, bb, pa);
    LookWord<k64, kClean>(g, v0.w, bn, pn, pa, t.base, f);
    LookProbe<k64, 0, kClean>(v1.y, t.base, f, bn, pn);
    LookWord<k64, kClean>(g, v1.x, bb, pa, pn, t.base, f);
    LookProbe<k64, 0, kClean>(v1.z, t.base, f, bb, pa);
    LookWord<k64, kClean>(g, v1.y, bn, pn, pa, t.base, f);
    LookProbe<k64, 0, kClean>(v1.w, t.base, f, bn, pn);
    LookWord<k64, kClean>(g, v1.z, bb, pa, pn, t.base, f);
    LookProbe<k64, 0, kClean>(late(g), t.base, f, bb, pa);
    LookWord<k64, kClean>(g, v1.w, bn, pn, more ? pa : (kClean ? 0x80000000u : 0xffffffffu), t.base, f);
    if (g == t.H) {
        prev = ReplayBlock32(args, prev, v0, v1);
        g = prev < t.H ? prev : t.H;
    }
}

// The word after the block was requested from HBM when this block began: its probe must stay down here (an ordinary
// intrinsic is hoisted to the top of the block by the compiler, where it waits for the whole DRAM latency).
// (a volatile mov is not enough: ptxas schedules across it.  The word is made to depend on the walk itself -- plus g
// times a kernel argument that is always zero -- which costs one IMAD per block.)
template <bool k64, bool kClean = false>
__device__ __forceinline__ void LookBlock32(const Tables& t, uint32_t& g, uint32_t& prev, const uint4& v0, const uint4& v1,
                                            uint32_t next0, bool more, const LookFilter& f, uint32_t opaque_zero, const ScanArgs* args)
{
    LookBlock32<k64, kClean>(t, g, prev, v0, v1, more, f, [=](uint32_t g) { return next0 + g * opaque_zero; }, args);
}

// Register budget.  The register file is split between the four warp schedulers (16 K registers each), so a
// CTA's warps should be a multiple of four: 512 threads x 3 CTAs leaves 40 registers per thread (12 warps x 1280
// per scheduler), 384 threads x 3 CTAs or 640 threads x 2 CTAs leave 48 (9 / 10 warps x 1536).  The kernel is short
// of independent chains, so it runs the ten-warp shape at 48 registers.
constexpr int kLookBlock48 = 640;

template <bool k64, int kRegs, bool kClean, bool kStarts>
__global__ void __maxnreg__(kRegs) ScanUniformLookKernel(const __grid_constant__ ScanArgs a)
{
    uint8_t* const smem = pire_b200_smem;
    SharedView sv = CarveShared(smem, a.hot);
    StageTables(a, sv, a.hot8, a.hot);

    Tables t;
    t.hot = sv.hot;
    t.base = SmemWindowBase();          // the hot rows are the first thing in the array (CarveShared, no private region)
    t.cls = sv.cls;
    t.full = a.full;
    t.H = a.hot;
    t.letters = a.letters;
    t.wide = a.wide;
    t.m0 = a.look_bitmap;
    LookFilter f;
    f.lo = k64 ? (uint32_t) a.look_bitmap64 : a.look_bitmap;
    f.hi = (uint32_t) (a.look_bitmap64 >> 32);
    f.zero = a.opaque_zero;
    f.rev = __brev(f.lo);

    const uint32_t units = (uint32_t) ((a.n + 31) / 32);            // pire_gpu_run_batch keeps n <= 2^40: units below 2^32
    const uint32_t warps_per_block = blockDim.x >> 5;
    const uint32_t warps = gridDim.x * warps_per_block;
    const uint32_t len = (uint32_t) a.fixed_len;
    const uint32_t blocks = len >> 5;                               // 32-byte blocks per string (uniform)

    for (uint32_t unit = blockIdx.x * warps_per_block + (threadIdx.x >> 5); unit < units; unit += warps) {
        uint32_t g, prev;
        bool known;
        {
            const uint64_t i = (uint64_t) unit * 32 + (threadIdx.x & 31);
            const uint8_t* p = a.corpus + (i < a.n ? i : a.n - 1) * (uint64_t) len;
            const uint32_t start = LaneStart<kStarts>(a, t, i, i < a.n, known);
            prev = start;
            g = start < t.H ? start : t.H;
            if (blocks != 0) {
                uint4 a0, a1, b0, b1;
                LoadStream32(p, a0, a1);
                for (uint32_t left = blocks;;) {
                    // `left` counts the blocks not yet walked, the one in the a-set included
                    const bool more_b = left > 1;
                    p += 32;
                    if (more_b)
                        LoadStream32(p, b0, b1);
                    __syncwarp();          // see below
                    LookBlock32<k64, kClean>(t, g, prev, a0, a1, b0.x, more_b, f, a.opaque_zero, &a);
                    if (!more_b)
                        break;
                    const bool more_a = left > 2;
                    p += 32;
                    if (more_a)
                        LoadStream32(p, a0, a1);
                    // The warp barrier pins the loads HERE.  Left alone, the scheduler sinks the two LDG.128 towards
                    // their first use to lend their eight destination registers to the steps in between, which exposes
                    // most of a DRAM round trip per block (long-scoreboard waits on the first use of the loaded word).
                    __syncwarp();
                    LookBlock32<k64, kClean>(t, g, prev, b0, b1, a0.x, more_a, f, a.opaque_zero, &a);
                    left -= 2;
                    // multi.h:955-958,:979-982 (NoExit), looked at every 64 bytes here
                    if (!more_a || __all_sync(0xffffffffu, sv.noexit[g] != 0))
                        break;
                }
            }
        }
        const uint64_t i = (uint64_t) unit * 32 + (threadIdx.x & 31);
        LaneState s;
        s.g = t.H;              // Report reads the complete state
        s.cold = g == t.H ? prev : g;
        Report(a, t, s, unit, i, i < a.n, known);
    }
}

// ---------------------------------------------------------------- LOOK variant, two strings per lane
//
// The one-string look-ahead kernel waits mostly on the LOP3 that needs the previous step's LDS, and more warps per SM
// run it faster -- it is short of independent chains, and registers (48 per thread) cap the warps.  Here every lane walks TWO strings (units 2p and 2p+1 of the
// batch) step by step in turn: the second string's step fills the latency of the first one's table read, and the
// block bookkeeping is shared.
template <bool kClean>
__device__ __forceinline__ void LookWord2(uint32_t& ga, uint32_t wa, uint32_t bba0, uint32_t paa0, uint32_t pana, uint32_t& gb, uint32_t wb,
                                          uint32_t bbb0, uint32_t pab0, uint32_t panb, uint32_t base, const LookFilter& f)
{
    uint32_t bba1, bba2, bba3, paa1, paa2, paa3, bbb1, bbb2, bbb3, pab1, pab2, pab3;
    LookProbe<false, 1, kClean>(wa, base, f, bba1, paa1);
    LookProbe<false, 1, kClean>(wb, base, f, bbb1, pab1);
    LookStep<kClean>(ga, bba0, paa0, paa1);
    LookStep<kClean>(gb, bbb0, pab0, pab1);
    LookProbe<false, 2, kClean>(wa, base, f, bba2, paa2);
    LookProbe<false, 2, kClean>(wb, base, f, bbb2, pab2);
    LookStep<kClean>(ga, bba1, paa1, paa2);
    LookStep<kClean>(gb, bbb1, pab1, pab2);
    LookProbe<false, 3, kClean>(wa, base, f, bba3, paa3);
    LookProbe<false, 3, kClean>(wb, base, f, bbb3, pab3);
    LookStep<kClean>(ga, bba2, paa2, paa3);
    LookStep<kClean>(gb, bbb2, pab2, pab3);
    LookStep<kClean>(ga, bba3, paa3, pana);
    LookStep<kClean>(gb, bbb3, pab3, panb);
}

// `late(ga, gb, latea, lateb)` fetches the first words of the blocks that follow, after the walk of the block's first 28
// bytes (see LookBlock32), from the ring in shared memory (ScanUniformLookRingKernel).
template <bool kClean, typename Late>
__device__ __forceinline__ void LookBlock32x2(const Tables& t, uint32_t& ga, uint32_t& preva, const uint4& a0, const uint4& a1,
                                              uint32_t& gb, uint32_t& prevb, const uint4& b0, const uint4& b1, bool more,
                                              const LookFilter& f, Late late, const ScanArgs* args)
{
    preva = ga == t.H ? preva : ga;
    prevb = gb == t.H ? prevb : gb;
    uint32_t bba, paa, bna, pna, bbb, pab, bnb, pnb;
    LookProbe<false, 0, kClean>(a0.x, t.base, f, bba, paa);
    LookProbe<false, 0, kClean>(b0.x, t.base, f, bbb, pab);
    LookProbe<false, 0, kClean>(a0.y, t.base, f, bna, pna);
    LookProbe<false, 0, kClean>(b0.y, t.base, f, bnb, pnb);
    LookWord2<kClean>(ga, a0.x, bba, paa, pna, gb, b0.x, bbb, pab, pnb, t.base, f);
    LookProbe<false, 0, kClean>(a0.z, t.base, f, bba, paa);
    LookProbe<false, 0, kClean>(b0.z, t.base, f, bbb, pab);
    LookWord2<kClean>(ga, a0.y, bna, pna, paa, gb, b0.y, bnb, pnb, pab, t.base, f);
    LookProbe<false, 0, kClean>(a0.w, t.base, f, bna, pna);
    LookProbe<false, 0, kClean>(b0.w, t.base, f, bnb, pnb);
    LookWord2<kClean>(ga, a0.z, bba, paa, pna, gb, b0.z, bbb, pab, pnb, t.base, f);
    LookProbe<false, 0, kClean>(a1.x, t.base, f, bba, paa);
    LookProbe<false, 0, kClean>(b1.x, t.base, f, bbb, pab);
    LookWord2<kClean>(ga, a0.w, bna, pna, paa, gb, b0.w, bnb, pnb, pab, t.base, f);
    LookProbe<false, 0, kClean>(a1.y, t.base, f, bna, pna);
    LookProbe<false, 0, kClean>(b1.y, t.base, f, bnb, pnb);
    LookWord2<kClean>(ga, a1.x, bba, paa, pna, gb, b1.x, bbb, pab, pnb, t.base, f);
    LookProbe<false, 0, kClean>(a1.z, t.base, f, bba, paa);
    LookProbe<false, 0, kClean>(b1.z, t.base, f, bbb, pab);
    LookWord2<kClean>(ga, a1.y, bna, pna, paa, gb, b1.y, bnb, pnb, pab, t.base, f);
    LookProbe<false, 0, kClean>(a1.w, t.base, f, bna, pna);
    LookProbe<false, 0, kClean>(b1.w, t.base, f, bnb, pnb);
    LookWord2<kClean>(ga, a1.z, bba, paa, pna, gb, b1.z, bbb, pab, pnb, t.base, f);
    // the words after the blocks are still on their way from HBM: their probes stay behind the walk (see LookBlock32)
    uint32_t latea, lateb;
    late(ga, gb, latea, lateb);
    LookProbe<false, 0, kClean>(latea, t.base, f, bba, paa);
    LookProbe<false, 0, kClean>(lateb, t.base, f, bbb, pab);
    LookWord2<kClean>(ga, a1.w, bna, pna, more ? paa : 0x80000000u, gb, b1.w, bnb, pnb, more ? pab : 0x80000000u, t.base, f);
    if (ga == t.H) {
        preva = ReplayBlock32(args, preva, a0, a1);
        ga = preva < t.H ? preva : t.H;
    }
    if (gb == t.H) {
        prevb = ReplayBlock32(args, prevb, b0, b1);
        gb = prevb < t.H ? prevb : t.H;
    }
}

// ---------------------------------------------------------------- LOOK variant, two strings per lane, fed from a ring
//
// Two strings per lane fed from registers, one 32-byte block of each string in flight (a kernel since removed), moved
// about half of what HBM can deliver: the scan is bound by its loads, not by the walk.  More blocks in flight per string
// would take registers such a kernel does not have, so here each lane copies its blocks with cp.async (LDGSTS) into a private ring in
// shared memory, three slots per string, and reads a block into registers (two LDS.128 per string) only when it walks
// it: two blocks of each string are on their way while one is walked.  Same walk, same pairs of units, same NoExit exit
// every 64 bytes; one CTA of 24 warps per SM.  The shape is the fastest of the ring shapes tools/microbench.cu measures
// without the walk (DESIGN.md section 4): 24 warps x 3 slots beat 28 x 2 and 32 x 2.
// A slot of a warp is two 512-byte rows, one per 16-byte half, so the copies and the reads of a warp are free of bank
// conflicts: per warp, slot k of string s (0, 1) sits at k * 2048 + s * 1024, its second half 512 bytes further.
constexpr int kRingBlock = 768;
constexpr uint32_t kRingSlots = 3;
constexpr uint32_t kRingSlotBytes = 2048;
constexpr size_t kRingWarpBytes = (size_t) kRingSlots * kRingSlotBytes;      // 6 KB; 144 KB per CTA beside <= 75.5 KB of tables

__device__ __forceinline__ uint32_t NextSlot(uint32_t slot) { return slot + kRingSlotBytes == kRingWarpBytes ? 0 : slot + kRingSlotBytes; }

// One 32-byte block of a string into its slot.  cp.async.cg: both 16-byte halves go to L2, which in the ring measured
// faster than .ca (the register loads are the other way round); the first half carries the 128-byte L2 prefetch-size
// hint of LoadStream32, so that an L2 miss fetches the line that holds the string's next three blocks.
__device__ __forceinline__ void CopyBlock32(uint32_t dst_shared, const uint8_t* src)
{
    asm volatile("cp.async.cg.shared.global.L2::128B [%0], [%1], 16;\n\t"
                 "cp.async.cg.shared.global [%2], [%3], 16;" ::"r"(dst_shared), "l"(src), "r"(dst_shared + 512), "l"(src + 16)
                 : "memory");
}

__device__ __forceinline__ uint32_t LoadShared4(uint32_t shared_addr)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(shared_addr) : "memory");
    return v;
}

// The first words of the next blocks, read after the walk of this block's first 28 bytes once their commit group has
// landed.  The address depends on the walk (plus g times a kernel argument that is always zero), so the read cannot be
// hoisted to where the copy may still be in flight.
struct RingNext {
    uint32_t at;          // the next block's slot, string a; string b 1024 bytes further
    uint32_t zero;
    __device__ __forceinline__ void operator()(uint32_t ga, uint32_t gb, uint32_t& latea, uint32_t& lateb) const
    {
        CopyAsyncWait<kRingSlots - 1>();
        latea = LoadShared4(at + ga * zero);
        lateb = LoadShared4(at + 1024 + gb * zero);
    }
};

// The walk of ScanUniformLookRingKernel, and with kStarts of ScanUniformLookRingFromKernel (each string from its own start).
template <bool kStarts>
__device__ __forceinline__ void LookRingScan(const ScanArgs& a)
{
    uint8_t* const smem = pire_b200_smem;
    SharedView sv = CarveShared(smem, a.hot);
    StageTables(a, sv, a.hot8, a.hot);

    Tables t;
    t.hot = sv.hot;
    t.base = SmemWindowBase();
    t.cls = sv.cls;
    t.full = a.full;
    t.H = a.hot;
    t.letters = a.letters;
    t.wide = a.wide;
    t.m0 = a.look_bitmap;
    LookFilter f;
    f.lo = a.look_bitmap;
    f.hi = 0;
    f.zero = a.opaque_zero;
    f.rev = __brev(f.lo);

    const uint32_t units = (uint32_t) ((a.n + 31) / 32);
    const uint32_t pairs = (units + 1) / 2;
    const uint32_t warps_per_block = blockDim.x >> 5;
    const uint32_t warps = gridDim.x * warps_per_block;
    const uint32_t len = (uint32_t) a.fixed_len;
    const uint32_t blocks = len >> 5;
    // this lane's 16-byte column of its warp's ring (slot 0, string a, first half)
    const uint32_t ring = SmemAddr(sv.stage) + (threadIdx.x >> 5) * (uint32_t) kRingWarpBytes + (threadIdx.x & 31) * 16;

    for (uint32_t pair = blockIdx.x * warps_per_block + (threadIdx.x >> 5); pair < pairs; pair += warps) {
        const bool second = 2 * pair + 1 < units;          // the last pair of an odd batch walks its first unit twice
        uint32_t ga, preva, gb, prevb;
        bool knowna, knownb;
        {
            const uint64_t ia = (uint64_t) pair * 64 + (threadIdx.x & 31);
            const uint64_t ib = ia + (second ? 32 : 0);
            const uint8_t* pa = a.corpus + (ia < a.n ? ia : a.n - 1) * (uint64_t) len;
            const uint8_t* pb = a.corpus + (ib < a.n ? ib : a.n - 1) * (uint64_t) len;
            if constexpr (kStarts) {
                preva = LaneStart<true>(a, t, ia, ia < a.n, knowna);
                prevb = LaneStart<true>(a, t, ib, ib < a.n, knownb);
                ga = preva < t.H ? preva : t.H;
                gb = prevb < t.H ? prevb : t.H;
            } else {
                // as it was before starts existed: the kernel compiles to the same code
                knowna = knownb = true;
                preva = prevb = a.start;
                ga = gb = a.start < t.H ? a.start : t.H;
            }
            if (blocks != 0) {
                // Blocks 0..2 of both strings, one commit group per block (empty past the end); block k + 3 refills the
                // slot of block k as soon as block k is in registers.  No copy reaches past the end of a string: the
                // last string of a batch may end where its allocation ends.
#pragma unroll
                for (uint32_t j = 0; j < kRingSlots; ++j) {
                    if (j < blocks) {
                        CopyBlock32(ring + j * kRingSlotBytes, pa + 32 * j);
                        CopyBlock32(ring + j * kRingSlotBytes + 1024, pb + 32 * j);
                    }
                    CopyAsyncCommit();
                }
                CopyAsyncWait<kRingSlots - 1>();                    // block 0 has landed
                uint32_t s0 = 0;                                    // slot of block k
                for (uint32_t k = 0;; k += 2) {
                    // block k (landed: the prologue's wait or the previous block's late one)
                    const uint32_t s1 = NextSlot(s0);
                    uint4 a0 = LoadShared16(ring + s0), a1 = LoadShared16(ring + s0 + 512);
                    uint4 b0 = LoadShared16(ring + s0 + 1024), b1 = LoadShared16(ring + s0 + 1536);
                    if (k + kRingSlots < blocks) {
                        CopyBlock32(ring + s0, pa + 32 * (size_t) (k + kRingSlots));
                        CopyBlock32(ring + s0 + 1024, pb + 32 * (size_t) (k + kRingSlots));
                    }
                    CopyAsyncCommit();
                    const bool more_1 = k + 1 < blocks;
                    LookBlock32x2<true>(t, ga, preva, a0, a1, gb, prevb, b0, b1, more_1, f, RingNext{ring + s1, a.opaque_zero}, &a);
                    if (!more_1)
                        break;
                    // block k + 1
                    const uint32_t s2 = NextSlot(s1);
                    a0 = LoadShared16(ring + s1), a1 = LoadShared16(ring + s1 + 512);
                    b0 = LoadShared16(ring + s1 + 1024), b1 = LoadShared16(ring + s1 + 1536);
                    if (k + 1 + kRingSlots < blocks) {
                        CopyBlock32(ring + s1, pa + 32 * (size_t) (k + 1 + kRingSlots));
                        CopyBlock32(ring + s1 + 1024, pb + 32 * (size_t) (k + 1 + kRingSlots));
                    }
                    CopyAsyncCommit();
                    const bool more_2 = k + 2 < blocks;
                    LookBlock32x2<true>(t, ga, preva, a0, a1, gb, prevb, b0, b1, more_2, f, RingNext{ring + s2, a.opaque_zero}, &a);
                    // multi.h:955-958,:979-982 (NoExit), looked at every 64 bytes
                    if (!more_2 || __all_sync(0xffffffffu, (sv.noexit[ga] & sv.noexit[gb]) != 0))
                        break;
                    s0 = s2;
                }
                CopyAsyncWait<0>();            // a NoExit exit leaves copies in flight: they land before the slots are reused
            }
        }
        const uint64_t ia = (uint64_t) pair * 64 + (threadIdx.x & 31);
        LaneState s;
        s.g = t.H;
        s.cold = ga == t.H ? preva : ga;
        Report(a, t, s, 2 * (uint64_t) pair, ia, ia < a.n, knowna);
        if (second) {
            s.cold = gb == t.H ? prevb : gb;
            Report(a, t, s, 2 * (uint64_t) pair + 1, ia + 32, ia + 32 < a.n, knownb);
        }
    }
}

__global__ void __launch_bounds__(kRingBlock, 1) ScanUniformLookRingKernel(const __grid_constant__ ScanArgs a) { LookRingScan<false>(a); }

// The same kernel with per-string starts (pire_gpu_run_batch_from), under a name of its own: the one above is the one
// that runs without.
__global__ void __launch_bounds__(kRingBlock, 1) ScanUniformLookRingFromKernel(const __grid_constant__ ScanArgs a) { LookRingScan<true>(a); }

// ---------------------------------------------------------------- LOOK variant, one string per lane, fed from a ring
//
// Two strings per lane were made for the register-fed kernel, which was short of independent chains and of registers.
// With the input in a ring the registers are free again: a one-string walk needs one block's eight data registers and
// the late word, so 32 warps fit in one CTA.  Here each lane walks one string (ScanUniformLookKernel's walk: 32-slot
// filter, clean probes) from a ring of kSlots blocks; kSlots - 1 blocks of every string are on their way while one is
// walked, and half as many lines are in progress in L2 as with two strings per lane.  NoExit exit every 64 bytes, as in
// the other look-ahead kernels.  The shape, one CTA of 32 warps per SM with three slots (96 KB of ring), is the fastest
// of the walk at 16 x 8, 24 x 6, 28 x 5, 32 x 3 and 32 x 4 (DESIGN.md section 4): fewer warps starve the walk of
// chains even where their loads alone run faster.  A slot of a warp is two 512-byte rows, one per 16-byte half, so the
// copies and the reads of a warp are free of bank conflicts: per warp, slot k sits at k * 1024.
constexpr int kRing1Block = 1024;
constexpr int kRing1Slots = 3;
constexpr uint32_t kRing1SlotBytes = 1024;
template <int kSlots>
__device__ __forceinline__ uint32_t NextSlot1(uint32_t slot) { return slot + kRing1SlotBytes == kSlots * kRing1SlotBytes ? 0 : slot + kRing1SlotBytes; }

// The first word of the next block, read after the walk of this block's first 28 bytes once its commit group has landed;
// the address depends on the walk, as in RingNext.
template <int kSlots>
struct RingNext1 {
    uint32_t at;          // the next block's slot
    uint32_t zero;
    __device__ __forceinline__ uint32_t operator()(uint32_t g) const
    {
        CopyAsyncWait<kSlots - 1>();
        return LoadShared4(at + g * zero);
    }
};

template <int kSlots, bool kStarts>
__global__ void __launch_bounds__(kRing1Block, 1) ScanUniformLookRing1Kernel(const __grid_constant__ ScanArgs a)
{
    uint8_t* const smem = pire_b200_smem;
    SharedView sv = CarveShared(smem, a.hot);
    StageTables(a, sv, a.hot8, a.hot);

    Tables t;
    t.hot = sv.hot;
    t.base = SmemWindowBase();
    t.cls = sv.cls;
    t.full = a.full;
    t.H = a.hot;
    t.letters = a.letters;
    t.wide = a.wide;
    t.m0 = a.look_bitmap;
    LookFilter f;
    f.lo = a.look_bitmap;
    f.hi = 0;
    f.zero = a.opaque_zero;
    f.rev = __brev(f.lo);

    const uint32_t units = (uint32_t) ((a.n + 31) / 32);
    const uint32_t warps_per_block = blockDim.x >> 5;
    const uint32_t warps = gridDim.x * warps_per_block;
    const uint32_t len = (uint32_t) a.fixed_len;
    const uint32_t blocks = len >> 5;
    // this lane's 16-byte column of its warp's ring (slot 0, first half)
    const uint32_t ring = SmemAddr(sv.stage) + (threadIdx.x >> 5) * (uint32_t) (kSlots * kRing1SlotBytes) + (threadIdx.x & 31) * 16;

    for (uint32_t unit = blockIdx.x * warps_per_block + (threadIdx.x >> 5); unit < units; unit += warps) {
        uint32_t g, prev;
        bool known;
        {
            const uint64_t i = (uint64_t) unit * 32 + (threadIdx.x & 31);
            const uint8_t* p = a.corpus + (i < a.n ? i : a.n - 1) * (uint64_t) len;
            const uint32_t start = LaneStart<kStarts>(a, t, i, i < a.n, known);
            prev = start;
            g = start < t.H ? start : t.H;
            if (blocks != 0) {
                // Blocks 0..kSlots-1, one commit group per block (empty past the end); block k + kSlots refills the slot
                // of block k as soon as block k is in registers.  No copy reaches past the end of a string: the last
                // string of a batch may end where its allocation ends.
#pragma unroll
                for (uint32_t j = 0; j < kSlots; ++j) {
                    if (j < blocks)
                        CopyBlock32(ring + j * kRing1SlotBytes, p + 32 * j);
                    CopyAsyncCommit();
                }
                CopyAsyncWait<kSlots - 1>();                        // block 0 has landed
                uint32_t s0 = 0;                                    // slot of block k
                for (uint32_t k = 0;; k += 2) {
                    // block k (landed: the prologue's wait or the previous block's late one)
                    const uint32_t s1 = NextSlot1<kSlots>(s0);
                    uint4 v0 = LoadShared16(ring + s0), v1 = LoadShared16(ring + s0 + 512);
                    if (k + kSlots < blocks)
                        CopyBlock32(ring + s0, p + 32 * (size_t) (k + kSlots));
                    CopyAsyncCommit();
                    const bool more_1 = k + 1 < blocks;
                    LookBlock32<false, true>(t, g, prev, v0, v1, more_1, f, RingNext1<kSlots>{ring + s1, a.opaque_zero}, &a);
                    if (!more_1)
                        break;
                    // block k + 1
                    const uint32_t s2 = NextSlot1<kSlots>(s1);
                    v0 = LoadShared16(ring + s1), v1 = LoadShared16(ring + s1 + 512);
                    if (k + 1 + kSlots < blocks)
                        CopyBlock32(ring + s1, p + 32 * (size_t) (k + 1 + kSlots));
                    CopyAsyncCommit();
                    const bool more_2 = k + 2 < blocks;
                    LookBlock32<false, true>(t, g, prev, v0, v1, more_2, f, RingNext1<kSlots>{ring + s2, a.opaque_zero}, &a);
                    // multi.h:955-958,:979-982 (NoExit), looked at every 64 bytes
                    if (!more_2 || __all_sync(0xffffffffu, sv.noexit[g] != 0))
                        break;
                    s0 = s2;
                }
                CopyAsyncWait<0>();            // a NoExit exit leaves copies in flight: they land before the slots are reused
            }
        }
        const uint64_t i = (uint64_t) unit * 32 + (threadIdx.x & 31);
        LaneState s;
        s.g = t.H;
        s.cold = g == t.H ? prev : g;
        Report(a, t, s, unit, i, i < a.n, known);
    }
}

// Edge chunk of a string (its first or last, partially owned 16 bytes): loaded once, then
// handed out byte by byte from registers.
__device__ __forceinline__ uint4 LoadEdge16(const uint8_t* aligned)
{
    uint4 v;
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(aligned));
    return v;
}

struct EdgeBytes {
    uint64_t lo, hi;
    __device__ __forceinline__ EdgeBytes(uint4 v, uint32_t skip)
    {
        lo = (uint64_t) v.x | ((uint64_t) v.y << 32);
        hi = (uint64_t) v.z | ((uint64_t) v.w << 32);
        if (skip >= 8) {
            lo = hi;
            hi = 0;
            skip -= 8;
        }
        if (skip) {
            lo = (lo >> (8 * skip)) | (hi << (64 - 8 * skip));
            hi >>= 8 * skip;
        }
    }
    __device__ __forceinline__ uint32_t Next()
    {
        uint32_t b = (uint32_t) lo & 0xffu;
        lo = (lo >> 8) | (hi << 56);
        hi >>= 8;
        return b;
    }
    // the remaining bytes as four words, the next byte in bits 0-7 of .x
    __device__ __forceinline__ uint4 Words() const
    {
        return make_uint4((uint32_t) lo, (uint32_t) (lo >> 32), (uint32_t) hi, (uint32_t) (hi >> 32));
    }
};

// The first n (1..16) bytes of `v` through the hot rows: whole words with the fast step, the last one to
// three bytes one by one -- two to three instructions per byte instead of the slow step's compare, branch
// and table choice.  Short strings (lines of text) consist mostly of such edge bytes.  A lane that is, or
// ends up, outside the hot rows replays the bytes through the complete table.
template <bool kPred>
__device__ __forceinline__ void EdgeFast(const Tables& t, LaneState& s, uint4 v, uint32_t n)
{
    const uint32_t before = s.g;
    uint32_t g = before;
    const uint32_t words = n >> 2, rest = n & 3;
    if (words > 0)
        FastWord<kPred>(t, g, v.x);
    if (words > 1)
        FastWord<kPred>(t, g, v.y);
    if (words > 2)
        FastWord<kPred>(t, g, v.z);
    if (words > 3)
        FastWord<kPred>(t, g, v.w);
    const uint32_t last = words == 0 ? v.x : words == 1 ? v.y : words == 2 ? v.z : v.w;
    if (rest > 0)
        FastStep<kPred>(t, g, last, 0x5540);
    if (rest > 1)
        FastStep<kPred>(t, g, last, 0x5541);
    if (rest > 2)
        FastStep<kPred>(t, g, last, 0x5542);
    s.g = g;
    if (g == t.H) {
        uint32_t full = before == t.H ? s.cold : before;
        EdgeBytes eb(v, 0);
        for (uint32_t k = 0; k < n; ++k)
            full = SlowStep(t, full, eb.Next());
        SetFull(t, s, full);
    }
}

// An aligned 16-byte chunk that may stick out of the caller's buffer at either end (the very first and the
// very last chunk of a corpus): bytes outside read as zero.  Out of line, it is rare.
__device__ __noinline__ uint4 LoadEdge16Clipped(const uint8_t* aligned, uintptr_t buf_lo, uintptr_t buf_hi)
{
    uint32_t w[4] = {0, 0, 0, 0};
    for (int k = 0; k < 16; ++k) {
        const uintptr_t at = reinterpret_cast<uintptr_t>(aligned) + k;
        if (at >= buf_lo && at < buf_hi)
            w[k >> 2] |= (uint32_t) aligned[k] << (8 * (k & 3));
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

__device__ __forceinline__ uint4 LoadChunk16(const uint8_t* aligned, uintptr_t buf_lo, uintptr_t buf_hi)
{
    if (reinterpret_cast<uintptr_t>(aligned) >= buf_lo && reinterpret_cast<uintptr_t>(aligned) + 16 <= buf_hi)
        return LoadEdge16(aligned);
    return LoadEdge16Clipped(aligned, buf_lo, buf_hi);
}

// Generic batch: CSR offsets or arbitrary fixed length / alignment.  Head and
// tail bytes (to 16-byte alignment) take the slow step, like run.h:186-226 does
// with its word-aligned body.
// The look-ahead filter of the LOOK variant (see LookStep) inside one 16-byte chunk of a CSR string: byte k reads the
// table only if bytes k and k+1 both pass; the chunk's last byte is filtered alone, so the lane's state is exact at
// every chunk boundary (edges, replays and the NoExit test see true states).
__device__ __forceinline__ void Chunk16Look(const Tables& t, LaneState& s, uint4 v, const LookFilter& f)
{
    const uint32_t before = s.g;
    uint32_t g = s.g;
    uint32_t bb, pa, bn, pn;
    LookProbe<false, 0>(v.x, t.base, f, bb, pa);
    LookProbe<false, 0>(v.y, t.base, f, bn, pn);
    LookWord<false>(g, v.x, bb, pa, pn, t.base, f);
    LookProbe<false, 0>(v.z, t.base, f, bb, pa);
    LookWord<false>(g, v.y, bn, pn, pa, t.base, f);
    LookProbe<false, 0>(v.w, t.base, f, bn, pn);
    LookWord<false>(g, v.z, bb, pa, pn, t.base, f);
    LookWord<false>(g, v.w, bn, pn, 0xffffffffu, t.base, f);
    s.g = g;
    if (g == t.H) {
        uint32_t from = before == t.H ? s.cold : before;
        uint32_t full = ReplayChunk(t.hot, t.cls, t.full, t.H, t.letters | (t.wide << 31), from, v);
        SetFull(t, s, full);
    }
}

// kMode: 0 plain, 1 exit filter (PRED), 2 exit filter with one byte of look-ahead (LOOK) in the 16-byte body chunks
template <int kMode, bool kStarts>
__global__ void __launch_bounds__(kBlock, kGenericBlocksPerSM) ScanGenericKernel(const __grid_constant__ ScanArgs a)
{
    constexpr bool kPred = kMode != 0;
    LookFilter look;
    look.lo = a.look_bitmap;
    look.hi = 0;
    look.zero = 0;
    look.rev = 0;
    uint8_t* const smem = pire_b200_smem;
    SharedView sv = CarveShared(smem, a.hot);
    StageTables(a, sv, a.hot8, a.hot);

    Tables t;
    t.hot = sv.hot;
    t.base = SmemAddr(sv.hot);
    t.cls = sv.cls;
    t.full = a.full;
    t.H = a.hot;
    t.letters = a.letters;
    t.wide = a.wide;
    t.m0 = a.exit_bitmap0;

    const uint32_t lane = threadIdx.x & 31;
    const uint64_t units = (a.n + 31) / 32;
    const uint64_t warps = (uint64_t) gridDim.x * kWarpsPerBlock;
    // staging ring: slot j of (warp w, lane l) at ((w * kStageSlots + j) * 32 + l) * 16 -- the 32
    // lanes of a warp read 512 contiguous bytes with one LDS.128 (conflict-free)
    const uint32_t stage = SmemAddr(sv.stage) + (((threadIdx.x >> 5) * kStageSlots) * 32 + lane) * 16;
    // [buf_lo, buf_hi): the caller's corpus buffer; whole aligned chunks may be read inside it only
    const uintptr_t buf_lo = reinterpret_cast<uintptr_t>(a.corpus);
    const uintptr_t buf_hi = buf_lo + (a.offsets ? a.offsets[a.n] - a.trim : a.n * a.fixed_len);
    const uint64_t split_first = a.split_count ? *a.split_count : 0;

    for (uint64_t unit = (uint64_t) blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);; unit += warps) {
        if (a.work_counter) {
            // length-binned launch: units are sorted longest first and claimed dynamically
            // (longest-processing-time-first keeps the 64 KiB strings off the tail)
            unsigned int claimed = 0;
            if (lane == 0)
                claimed = atomicAdd(a.work_counter, 1u);
            unit = __shfl_sync(0xffffffffu, claimed, 0);
        }
        if (unit >= units)
            break;
        const uint64_t slot = unit * 32 + lane;
        const bool valid = slot < a.n && slot >= split_first;          // the first split_first entries are the split kernel's
        const uint64_t i = valid && a.order ? a.order[slot] : slot;
        uint64_t b = 0, e = 0;
        if (valid) {
            if (a.offsets) {
                b = a.offsets[i];
                e = a.offsets[i + 1] - a.trim;
                e = e < b ? b : e;       // an empty entry of a trimmed (lines) batch, or caller offsets that step back
            } else {
                b = i * a.fixed_len;
                e = b + a.fixed_len;
            }
        }
        const uint8_t* p = a.corpus + b;
        const uint8_t* end = a.corpus + e;

        LaneState s;
        bool known;
        SetFull(t, s, LaneStart<kStarts>(a, t, i, valid, known));

        // head: up to the first 16-byte boundary.  The bytes come from ONE load of the aligned
        // chunk that holds them (the reference's RunChunk does the same with its head word,
        // run.h:129-151) instead of one dependent global load per byte; only a string whose edge
        // chunk would stick out of the corpus buffer reads its edge bytes one by one.
        {
            const uint32_t misalign = (uint32_t) (reinterpret_cast<uintptr_t>(p) & 15);
            if (p < end && misalign != 0) {
                const uint64_t room = (uint64_t) (end - p);
                const uint32_t nhead = room < 16 - misalign ? (uint32_t) room : 16 - misalign;
                const uint8_t* chunk = p - misalign;
                if (reinterpret_cast<uintptr_t>(chunk) >= buf_lo && reinterpret_cast<uintptr_t>(chunk) + 16 <= buf_hi) {
                    EdgeFast<kPred>(t, s, EdgeBytes(LoadEdge16(chunk), misalign).Words(), nhead);
                } else {
                    uint32_t full = FullState(t, s);
                    for (uint32_t k = 0; k < nhead; ++k)
                        full = SlowStep(t, full, p[k]);
                    SetFull(t, s, full);
                }
                p += nhead;
            }
        }
        // body: 16-byte chunks through a four-deep cp.async ring in shared memory (slot
        // c % 4 of this lane holds chunk c); the warp iterates until its longest lane is
        // done, shorter lanes idle (length binning keeps them few).
        const uint32_t chunks = (uint32_t) ((end - p) >> 4);
        bool parked = false;       // lane sits in a NoExit state: its remaining bytes are irrelevant
#pragma unroll
        for (int j = 0; j < kStageSlots; ++j) {
            if ((uint32_t) j < chunks)
                CopyAsync16(stage + j * 512, p + 16 * j);
            CopyAsyncCommit();
        }
        for (uint32_t k = 0; __any_sync(0xffffffffu, k < chunks); k += kStageSlots) {
#pragma unroll
            for (int j = 0; j < kStageSlots; ++j) {
                CopyAsyncWait<kStageSlots - 1>();                 // chunk k + j has landed
                const uint4 v = LoadShared16(stage + j * 512);
                if (k + kStageSlots + j < chunks)
                    CopyAsync16(stage + j * 512, p + 16 * (size_t) (k + kStageSlots + j));
                CopyAsyncCommit();
                if (k + j < chunks) {
                    if (kMode == 2)
                        Chunk16Look(t, s, v, look);
                    else
                        Chunk16<kPred>(t, s, v);
                }
            }
            // multi.h:955-958,:979-982: a NoExit state cannot be left by any byte.
            const bool live = k + kStageSlots < chunks;
            const bool stuck = sv.noexit[s.g] != 0;
            if (__all_sync(0xffffffffu, !live || stuck)) {
                parked = live && stuck;
                break;
            }
        }
        CopyAsyncWait<0>();
        // tail: fewer than 16 bytes, at an aligned address
        if (!parked) {
            p += 16 * (size_t) chunks;
            if (p < end) {
                const uint32_t ntail = (uint32_t) (end - p);
                if (reinterpret_cast<uintptr_t>(p) + 16 <= buf_hi) {
                    EdgeFast<kPred>(t, s, LoadEdge16(p), ntail);
                } else {
                    uint32_t full = FullState(t, s);
                    for (uint32_t k = 0; k < ntail; ++k)
                        full = SlowStep(t, full, p[k]);
                    SetFull(t, s, full);
                }
            }
        }
        if (a.order)
            ReportScattered(a, t, s, i, valid, known);
        else
            Report(a, t, s, unit, i, valid, known);
    }
}

// ---------------------------------------------------------------- long strings, split over a warp
//
// One string per lane makes the longest string of a batch the critical path: a 64 KiB string is 65 536 dependent
// table reads, milliseconds for a warp that shares its SM with 31 others -- as long as the whole mixed-length
// benchmark batch.  Here a WARP owns one long string: lane j walks piece j of 32 (whole 32-byte blocks,
// 32-byte loads one block ahead), lane 0 from the string's true state, the others from a guess (hot id 0, the most visited
// state).  Every lane leaves marks -- its hot id after every K blocks, in shared memory.  Then the pieces are stitched:
// lane j's true start is lane j-1's end; a lane whose walk started from another state re-walks its piece from the true
// one until it meets a mark (same hot id at the same position: the rest of the walk is the recorded one), replacing the
// marks it passes.  Two walks over the same bytes fall together within a few bytes for the automata regexps make (a
// byte that continues no match sends every state to the resting state), so a round of re-walks costs about K blocks;
// the loop repeats until every lane's start equals its predecessor's end, which is exact whatever the automaton does:
// lane 0 is exact, and lane j is exact one round after lane j-1 at the latest (31 rounds of a whole piece each in the
// worst case -- the serial walk).  A true start that is a NoExit state needs no walk at all.
constexpr uint32_t kSplitMin = 8192;            // bytes; a bucket boundary of LengthOrder
constexpr uint32_t kSplitMarks = 32;            // marks per lane
constexpr size_t kSplitMarkBytes = (size_t) kBlock * kSplitMarks;

__device__ __forceinline__ uint64_t EndOffset(const ScanArgs& a, uint64_t i)
{
    const uint64_t b = a.offsets[i], e = a.offsets[i + 1] - a.trim;
    return e < b ? b : e;
}

// One lane's piece of a split string: `my_blocks` whole 32-byte blocks at `piece`, walked from `s`, the hot id left in
// marks[32 * m] after every `per_mark` blocks.  Every lane runs the loop `trips` times (the longest piece of its warp),
// so that the scheduling fences behind the loads are reached by the whole warp.  The loads ask for the whole 256-byte
// line in L2: a piece is contiguous, seven of eight blocks then come from there.
template <bool kPred>
__device__ __forceinline__ void WalkPiece(const Tables& t, LaneState& s, const uint8_t* piece, uint32_t my_blocks, uint32_t trips,
                                          uint32_t per_mark, uint8_t* marks, uint32_t ahead)
{
    uint4 a0 = make_uint4(0, 0, 0, 0), a1 = a0, b0 = a0, b1 = a0;
    if (my_blocks)
        LoadStream32P(piece, a0, a1);
    uint32_t countdown = per_mark, m = 0;
    for (uint32_t k = 0; k < trips; k += 2) {
        // optional L2 prefetch, one per 256-byte line, `ahead` blocks in front of the walk.  The L2::256B hint
        // of the loads already brings the line into L2, so this was found to gain nothing.  Off by default.
        if (ahead && (k & 7u) == 0 && k + ahead < my_blocks)
            PrefetchL2(piece + 32 * (size_t) (k + ahead));
        if (k + 1 < my_blocks)
            LoadStream32P(piece + 32 * (size_t) (k + 1), b0, b1);
        __syncwarp();              // scheduling fence: the load is issued here, not next to its first use
        if (k < my_blocks) {
            Chunk16<kPred>(t, s, a0);
            Chunk16<kPred>(t, s, a1);
            if (--countdown == 0) {
                marks[32 * m++] = (uint8_t) s.g;
                countdown = per_mark;
            }
        }
        if (k + 2 < my_blocks)
            LoadStream32P(piece + 32 * (size_t) (k + 2), a0, a1);
        __syncwarp();
        if (k + 1 < my_blocks) {
            Chunk16<kPred>(t, s, b0);
            Chunk16<kPred>(t, s, b1);
            if (--countdown == 0) {
                marks[32 * m++] = (uint8_t) s.g;
                countdown = per_mark;
            }
        }
    }
}

// The piece again from its true start `want`, until the walk meets a mark (same hot id at the same place: from there
// on it is the recorded walk, and so is its end); marks passed on the way are replaced, so that they describe this
// walk afterwards.  Returns the piece's end state (`end_full` when a mark was met).  head0/head1 hold the piece's
// first block when head_fresh is set.
template <bool kPred>
__device__ __forceinline__ uint32_t RewalkPiece(const Tables& t, uint32_t want, const uint8_t* piece, uint32_t my_blocks,
                                                uint32_t per_mark, uint8_t* marks, uint4 head0, uint4 head1, bool& head_fresh,
                                                uint32_t end_full)
{
    LaneState r;
    SetFull(t, r, want);
    uint32_t countdown = per_mark, m = 0;
    bool met = false;
    uint4 v0 = head0, v1 = head1;
    if (!head_fresh && my_blocks)
        LoadStream32P(piece, v0, v1);
    head_fresh = false;
    for (uint32_t k = 0; k < my_blocks; ++k) {
        uint4 n0 = v0, n1 = v1;
        if (k + 1 < my_blocks)
            LoadStream32P(piece + 32 * (size_t) (k + 1), n0, n1);      // one block ahead, like the first walk
        Chunk16<kPred>(t, r, v0);
        Chunk16<kPred>(t, r, v1);
        if (--countdown == 0) {
            if (r.g != t.H && r.g == marks[32 * m]) {
                met = true;
                break;
            }
            marks[32 * m++] = (uint8_t) r.g;
            countdown = per_mark;
        }
        v0 = n0;
        v1 = n1;
    }
    return met ? end_full : FullState(t, r);
}

// The stitch of a warp's pieces: lane 0 must start from `first` (only lane 0's argument counts), every other lane where
// its predecessor ended.  A lane whose start changes walks its piece again (RewalkPiece); the loop repeats until no
// start changes, which is exact whatever the automaton does (lane j is exact one round after lane j-1 at the latest).
template <bool kPred>
__device__ __forceinline__ void StitchWarp(const Tables& t, const uint8_t* noexit, uint32_t first, uint32_t lane, const uint8_t* piece,
                                           uint32_t my_blocks, uint32_t per_mark, uint8_t* marks, uint4 head0, uint4 head1,
                                           bool& head_fresh, uint32_t& start_full, uint32_t& end_full)
{
    for (;;) {
        const uint32_t before = __shfl_up_sync(0xffffffffu, end_full, 1);
        const uint32_t want = lane == 0 ? first : before;
        const bool redo = want != start_full;
        if (!__any_sync(0xffffffffu, redo))
            break;
        if (redo) {
            start_full = want;
            const uint32_t n_marks = per_mark ? my_blocks / per_mark : 0u;
            if (want < t.H && noexit[want] != 0) {
                // multi.h:955-958: no byte leaves this state
                end_full = want;
                for (uint32_t m = 0; m < n_marks; ++m)
                    marks[32 * m] = (uint8_t) want;
            } else {
                end_full = RewalkPiece<kPred>(t, want, piece, my_blocks, per_mark, marks, head0, head1, head_fresh, end_full);
            }
        }
    }
}

// kStarts: the head and lane 0's piece start from the string's own start (LaneStart), the other pieces from the guess as
// ever; a start outside the scanner rides in bit 32 of the parked string number to the report.
template <bool kPred, bool kStarts>
__global__ void __launch_bounds__(kBlock, kMinBlocksPerSM) ScanSplitKernel(const __grid_constant__ ScanArgs a)
{
    uint8_t* const smem = pire_b200_smem;
    SharedView sv = CarveShared(smem, a.hot);
    StageTables(a, sv, a.hot8, a.hot);

    Tables t;
    t.hot = sv.hot;
    t.base = SmemAddr(sv.hot);
    t.cls = sv.cls;
    t.full = a.full;
    t.H = a.hot;
    t.letters = a.letters;
    t.wide = a.wide;
    t.m0 = a.exit_bitmap0;

    const uint32_t lane = threadIdx.x & 31;
    // mark m of lane l at marks[m * 32 + l]: the lanes of a warp write one mark with one conflict-free store
    uint8_t* const marks = sv.stage + (threadIdx.x >> 5) * (32 * kSplitMarks) + lane;
    volatile uint64_t* const parked = reinterpret_cast<volatile uint64_t*>(sv.stage + kSplitMarkBytes) + (threadIdx.x >> 5) * 4;
    const uintptr_t buf_lo = reinterpret_cast<uintptr_t>(a.corpus);
    const uintptr_t buf_hi = buf_lo + (a.offsets[a.n] - a.trim);
    const uint32_t n_long = *a.split_count;

    for (;;) {
        unsigned int slot = 0;
        if (lane == 0)
            slot = atomicAdd(a.split_counter, 1u);         // longest strings first
        slot = __shfl_sync(0xffffffffu, slot, 0);
        if (slot >= n_long)
            break;
        const uint64_t i = a.order[slot];
        const uint8_t* p = a.corpus + a.offsets[i];
        const uint8_t* const end = a.corpus + EndOffset(a, i);

        // head, by every lane alike: to the first 32-byte boundary
        LaneState s;
        bool known;
        SetFull(t, s, LaneStart<kStarts>(a, t, i, true, known));
        {
            const uint32_t mis = (uint32_t) (reinterpret_cast<uintptr_t>(p) & 15);
            if (p < end && mis != 0) {
                const uint64_t room = (uint64_t) (end - p);
                const uint32_t nhead = room < 16 - mis ? (uint32_t) room : 16 - mis;
                EdgeFast<kPred>(t, s, EdgeBytes(LoadChunk16(p - mis, buf_lo, buf_hi), mis).Words(), nhead);
                p += nhead;
            }
            if ((reinterpret_cast<uintptr_t>(p) & 16) && end - p >= 16) {
                Chunk16<kPred>(t, s, LoadEdge16(p));
                p += 16;
            }
        }
        const uint32_t blocks_total = (reinterpret_cast<uintptr_t>(p) & 31) ? 0u : (uint32_t) ((end - p) >> 5);
        const uint32_t base = blocks_total / 32, rem = blocks_total % 32;
        const uint32_t my_blocks = base + (lane < rem ? 1u : 0u);
        const uint32_t my_first = lane * base + (lane < rem ? lane : rem);
        const uint32_t trips = base + (rem ? 1u : 0u);                    // the longest piece
        const uint32_t per_mark = (trips + kSplitMarks - 1) / kSplitMarks;   // K: blocks between two marks (0 only if trips == 0)
        const uint8_t* const piece = p + 32 * (size_t) my_first;

        // the string's bounds wait in shared memory while the pieces are walked: they are the same in every lane and not
        // needed in the loop, which is short of registers (ptxas spilled the loop counter instead)
        if (lane == 0) {
            parked[0] = known ? i : i | (1ull << 32);          // i < 2^31
            parked[1] = reinterpret_cast<uint64_t>(p + 32 * (size_t) blocks_total);
            parked[2] = reinterpret_cast<uint64_t>(end);
        }
        __syncwarp();

        // the pieces, all at once: lane 0 from the string's state, the others from the guess
        uint32_t start_full = lane == 0 ? FullState(t, s) : 0u;
        SetFull(t, s, start_full);
        WalkPiece<kPred>(t, s, piece, my_blocks, trips, per_mark, marks, a.split_prefetch);
        uint32_t end_full = FullState(t, s);

        // A lane whose guess was wrong walks the head of its piece again: its first block is asked for now, before the
        // stitch knows who needs it (one 32-byte L2 hit per lane and string), so that the re-walk does not begin with a
        // bare load.
        uint4 head0 = make_uint4(0, 0, 0, 0), head1 = head0;
        bool head_fresh = my_blocks != 0;
        if (head_fresh)
            LoadStream32P(piece, head0, head1);

        // stitch: every lane must have started where its predecessor ended
        StitchWarp<kPred>(t, sv.noexit, start_full, lane, piece, my_blocks, per_mark, marks, head0, head1, head_fresh, start_full,
                          end_full);

        // tail, by every lane alike, from the last piece's end
        SetFull(t, s, __shfl_sync(0xffffffffu, end_full, 31));
        const uint8_t* q = reinterpret_cast<const uint8_t*>(parked[1]);
        const uint8_t* const q_end = reinterpret_cast<const uint8_t*>(parked[2]);
        if (q_end - q >= 16) {
            Chunk16<kPred>(t, s, LoadEdge16(q));
            q += 16;
        }
        if (q < q_end)
            EdgeFast<kPred>(t, s, LoadChunk16(q, buf_lo, buf_hi), (uint32_t) (q_end - q));
        const uint64_t at = parked[0];
        ReportScattered(a, t, s, kStarts ? (uint32_t) at : at, lane == 0, !kStarts || (at >> 32) == 0);
        __syncwarp();                      // the next string's bounds replace these
    }
}

// n_long = the number of leading entries of `order` whose strings are at least kSplitMin bytes long (LengthOrder puts the
// longest buckets first, so this is all of them; for any other permutation it is just some prefix, and the split kernel
// is exact for strings of any length).  Also resets the split kernel's work counter.
__global__ void SplitCountKernel(const uint64_t* __restrict__ offsets, const uint32_t* __restrict__ order, uint64_t n,
                                 uint32_t split_min, uint32_t* __restrict__ count, unsigned int* __restrict__ counter)
{
    if (threadIdx.x != 0 || blockIdx.x != 0)
        return;
    uint64_t lo = 0, hi = n;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        const uint64_t i = order[mid];
        if (offsets[i + 1] - offsets[i] >= split_min)
            lo = mid + 1;
        else
            hi = mid;
    }
    *count = (uint32_t) lo;
    *counter = 0;
}

// ---------------------------------------------------------------- one string over the whole grid
//
// The split kernel's walk lifted from a warp to the persistent grid (pire_gpu_run_string).  The 32-byte aligned body of
// the string is cut into one run of whole blocks per lane of the grid; the bytes before it (head) go to the grid's first
// lane, the bytes behind it (tail) to its last warp.  Every lane walks its piece from the guess (hot id 0) and leaves
// marks, only the first lane from the true state.  Then two levels of stitching:
//   1. inside a warp, StitchWarp as in the split kernel, with each warp's lane 0 keeping its own start;
//   2. across the grid, in rounds: every warp publishes its end (double-buffered, so that a round reads only what the
//      previous one wrote), grid.sync(), and every warp whose predecessor's end differs from its lane 0's start runs
//      StitchWarp again from that end and counts itself in the round's counter.  The rounds stop after one that
//      changes nothing.
// Exact whatever the automaton does: warp w is exact one round after warp w-1 at the latest.  Walks of regexp automata
// fall together within a few bytes, so the second round usually changes nothing; when they never do (parity of a run
// of a's) every round re-walks one warp's pieces and the grid degrades to the serial walk plus one grid.sync() per warp.
// A true start that is a NoExit state needs no walk at all.  Launched cooperatively (cudaLaunchCooperativeKernel):
// grid.sync() needs every CTA resident, and the grid never exceeds what the occupancy query allows.
constexpr int kStringBlocksPerSM = 2;           // 64 registers: the walk, the stitch and the rounds without spills
constexpr uint32_t kStringMinBlocks = 16;       // 32-byte blocks per lane below which the grid gets fewer CTAs

// Where the 32-byte aligned body of the string [p, end) begins: behind the bytes to the next 16-byte boundary and, if
// that is not a 32-byte one, 16 more.  A string too short for that has no body (the result is not 32-byte aligned).
__device__ __forceinline__ const uint8_t* StringBody(const uint8_t* p, const uint8_t* end)
{
    const uint32_t mis = (uint32_t) (reinterpret_cast<uintptr_t>(p) & 15);
    if (p < end && mis != 0)
        p += (uint64_t) (end - p) < 16 - mis ? (uint64_t) (end - p) : 16 - mis;
    if ((reinterpret_cast<uintptr_t>(p) & 16) && end - p >= 16)
        p += 16;
    return p;
}

// Both levels of the stitch for the lane's piece (`my_blocks` blocks at `piece`, walked from the guess by WalkPiece; the
// grid's first lane from first_start), in ScanStringKernel and CountStringKernel: StitchWarp inside the warp, then the
// rounds over the grid.  Ends after the last grid.sync() with start_full / end_full the true states at the start and at
// the end of the lane's piece.  A macro over the kernels' own variables, not a function: the same code as a
// __forceinline__ function changed ScanStringKernel's register allocation (8 bytes of spills), a macro leaves its SASS as
// it was.
#define PIRE_B200_STITCH_GRID(kPred)                                                                                           \
    do {                                                                                                                       \
        /* level 1: the warp's own pieces, lane 0 keeping its start */                                                         \
        StitchWarp<kPred>(t, sv.noexit, __shfl_sync(0xffffffffu, start_full, 0), lane, piece, my_blocks, per_mark, marks,      \
                          head0, head1, head_fresh, start_full, end_full);                                                     \
        if (lane == 31)                                                                                                        \
            __stcg(a.string_ends + warp, end_full);                                                                            \
        grid.sync();                                                                                                           \
        /* level 2: rounds over the grid.  Round r reads ends[(r-1) & 1], writes ends[r & 1] and counts its changes in       \
           counter[r % 3]; the counter of the next round is cleared in this one (its last readers finished two rounds ago) */ \
        for (uint32_t r = 1;; ++r) {                                                                                           \
            const uint32_t* const in = a.string_ends + ((r - 1) & 1) * warps;                                                  \
            uint32_t* const out = a.string_ends + (r & 1) * warps;                                                             \
            const uint32_t want = warp == 0 ? first_start : __ldcg(in + warp - 1);                                             \
            if (want != __shfl_sync(0xffffffffu, start_full, 0)) {                                                             \
                bool no_head = false; /* the prefetched first block served level 1; later rounds load it again */             \
                StitchWarp<kPred>(t, sv.noexit, want, lane, piece, my_blocks, per_mark, marks, make_uint4(0, 0, 0, 0),         \
                                  make_uint4(0, 0, 0, 0), no_head, start_full, end_full);                                      \
                if (lane == 0)                                                                                                 \
                    atomicAdd(a.string_rounds + r % 3, 1u);                                                                    \
            }                                                                                                                  \
            if (lane == 31)                                                                                                    \
                __stcg(out + warp, end_full);                                                                                  \
            if (me == 0)                                                                                                       \
                __stcg(a.string_rounds + (r + 1) % 3, 0u);                                                                     \
            grid.sync();                                                                                                       \
            if (__ldcg(a.string_rounds + r % 3) == 0)                                                                          \
                break;                                                                                                         \
        }                                                                                                                      \
    } while (0)

template <bool kPred>
__global__ void __launch_bounds__(kBlock, kStringBlocksPerSM) ScanStringKernel(const __grid_constant__ ScanArgs a)
{
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    uint8_t* const smem = pire_b200_smem;
    SharedView sv = CarveShared(smem, a.hot);
    StageTables(a, sv, a.hot8, a.hot);

    Tables t;
    t.hot = sv.hot;
    t.base = SmemAddr(sv.hot);
    t.cls = sv.cls;
    t.full = a.full;
    t.H = a.hot;
    t.letters = a.letters;
    t.wide = a.wide;
    t.m0 = a.exit_bitmap0;

    // the true start, in every thread alike: Initialize()[+Begin()] from the host, or the caller's StateIndex mapped to the
    // new numbering with BeginMark stepped here.  *a.start_idx may be the word the result goes to: it is written only
    // after a grid.sync(), when every thread has read it.
    uint32_t start = a.start;
    bool valid = true;
    if (a.start_idx)
        StartFrom(a, t, *a.start_idx, start, valid);
    const bool skip = !valid || (start < t.H && sv.noexit[start] != 0);       // multi.h:955-958: no byte leaves it

    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warp = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const uint32_t warps = gridDim.x * kWarpsPerBlock;
    uint8_t* const marks = sv.stage + (threadIdx.x >> 5) * (32 * kSplitMarks) + lane;
    const uintptr_t buf_lo = reinterpret_cast<uintptr_t>(a.corpus);
    const uintptr_t buf_hi = buf_lo + a.fixed_len;
    const uint8_t* p = a.corpus;
    const uint8_t* const end = a.corpus + a.fixed_len;

    // head, by the grid's first warp (all lanes alike): to the first 32-byte boundary
    LaneState s;
    SetFull(t, s, start);
    if (warp == 0 && !skip) {
        const uint32_t mis = (uint32_t) (buf_lo & 15);
        if (p < end && mis != 0) {
            const uint64_t room = (uint64_t) (end - p);
            const uint32_t nhead = room < 16 - mis ? (uint32_t) room : 16 - mis;
            EdgeFast<kPred>(t, s, EdgeBytes(LoadChunk16(p - mis, buf_lo, buf_hi), mis).Words(), nhead);
            p += nhead;
        }
        if ((reinterpret_cast<uintptr_t>(p) & 16) && end - p >= 16)
            Chunk16<kPred>(t, s, LoadEdge16(p));
    }
    p = StringBody(a.corpus, end);
    const uint32_t blocks_total = (reinterpret_cast<uintptr_t>(p) & 31) ? 0u : (uint32_t) ((end - p) >> 5);
    const uint32_t lanes = gridDim.x * kBlock;
    const uint32_t me = blockIdx.x * kBlock + threadIdx.x;
    const uint32_t base = blocks_total / lanes, rem = blocks_total % lanes;
    const uint32_t my_blocks = base + (me < rem ? 1u : 0u);
    const uint64_t my_first = (uint64_t) me * base + (me < rem ? me : rem);
    const uint32_t trips = base + (rem ? 1u : 0u);                    // the longest piece
    const uint32_t per_mark = (trips + kSplitMarks - 1) / kSplitMarks;   // blocks between two marks (0 only if trips == 0)
    const uint8_t* const piece = p + 32 * my_first;
    const uint32_t first_start = __shfl_sync(0xffffffffu, FullState(t, s), 0);   // warp 0: the state behind the head

    uint32_t start_full = me == 0 ? first_start : 0u;
    uint32_t end_full = start_full;
    if (!skip) {
        SetFull(t, s, start_full);
        WalkPiece<kPred>(t, s, piece, my_blocks, trips, per_mark, marks, 0);
        end_full = FullState(t, s);

        uint4 head0 = make_uint4(0, 0, 0, 0), head1 = head0;
        bool head_fresh = my_blocks != 0;
        if (head_fresh)
            LoadStream32P(piece, head0, head1);
        PIRE_B200_STITCH_GRID(kPred);
    } else {
        grid.sync();
    }
    if (warp != warps - 1)
        return;

    // tail, by the last warp (all lanes alike), from the last piece's end; the body's bounds again (cheaper than keeping
    // them in registers through the rounds)
    uint32_t last = start;
    if (!skip) {
        SetFull(t, s, __shfl_sync(0xffffffffu, end_full, 31));
        const uint8_t* q = StringBody(a.corpus, end);
        if ((reinterpret_cast<uintptr_t>(q) & 31) == 0)
            q += (size_t) (end - q) & ~(size_t) 31;
        if (end - q >= 16) {
            Chunk16<kPred>(t, s, LoadEdge16(q));
            q += 16;
        }
        if (q < end)
            EdgeFast<kPred>(t, s, LoadChunk16(q, buf_lo, buf_hi), (uint32_t) (end - q));
        last = FullState(t, s);
    }
    if (lane == 0) {
        // a start outside the scanner reads no table: match 0, mask 0, state 0xFFFFFFFF
        const DeviceFin f = valid ? a.fin[last] : DeviceFin{0u, 0u};
        if (a.match_bits)
            a.match_bits[0] = f.result >> 31;
        if (a.accept_masks)
            a.accept_masks[0] = f.mask;
        if (a.state_idx)
            a.state_idx[0] = valid ? f.result & 0x7fffffffu : 0xFFFFFFFFu;
    }
}

// ---------------------------------------------------------------- lines of text
//
// The step before the path for line-oriented input (samples/pigrep/pigrep.cpp:38-45): strings of a few dozen
// bytes of very unequal length (the reference's own benchmark prose: median 21 B, 90 % under 80 B, the longest
// of 32 consecutive lines 115 B on average).  One string per lane in lockstep units wastes three quarters of the
// lanes there -- each unit lasts as long as its longest line.  Here a warp owns 256 consecutive lines and its
// lanes pull them one at a time: every iteration each busy lane walks one aligned 16-byte chunk of its line
// (clipped to the line at both ends, fetched one chunk ahead into registers), and a lane that finishes reports
// its line and takes the next unassigned one (ballot + popcount over a warp-uniform cursor).  No staging ring:
// neighbouring lines share cache lines, so the chunks come from L1/L2.
constexpr uint32_t kLinesPerWarp = 256;
constexpr uint32_t kPiecesPerTurn = 2;      // chunks a busy lane walks before lines are handed out again
constexpr uint32_t kLinesMinIdle = 1;       // lanes that must be waiting before lines are handed out

template <bool kPred>
__global__ void __launch_bounds__(kBlock, kMinBlocksPerSM) ScanLinesKernel(const __grid_constant__ ScanArgs a)
{
    uint8_t* const smem = pire_b200_smem;
    SharedView sv = CarveShared(smem, a.hot);
    StageTables(a, sv, a.hot8, a.hot);

    Tables t;
    t.hot = sv.hot;
    t.base = SmemAddr(sv.hot);
    t.cls = sv.cls;
    t.full = a.full;
    t.H = a.hot;
    t.letters = a.letters;
    t.wide = a.wide;
    t.m0 = a.exit_bitmap0;

    const uint32_t lane = threadIdx.x & 31;
    const uint32_t below = (1u << lane) - 1u;
    const uint64_t groups = (a.n + kLinesPerWarp - 1) / kLinesPerWarp;
    const uint64_t warps = (uint64_t) gridDim.x * kWarpsPerBlock;
    const uintptr_t buf_lo = reinterpret_cast<uintptr_t>(a.corpus);
    const uintptr_t buf_hi = buf_lo + (a.offsets[a.n] - a.trim);

    for (uint64_t group = (uint64_t) blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5); group < groups; group += warps) {
        const uint64_t last = (group + 1) * kLinesPerWarp < a.n ? (group + 1) * kLinesPerWarp : a.n;
        uint64_t cursor = group * kLinesPerWarp;             // next unassigned line, the same in every lane
        bool busy = false;
        uint64_t line = 0;
        const uint8_t* chunk = a.corpus;
        uint32_t mis = 0, span = 0, pieces = 0, piece = 0;
        uint4 cur = make_uint4(0, 0, 0, 0);
        LaneState s;
        s.g = 0;
        s.cold = 0;
        for (;;) {
            const unsigned idle = __ballot_sync(0xffffffffu, !busy);
            // lines are handed out when enough lanes wait for one (or nobody is busy): handing out costs the
            // whole warp ~56 instructions however few lanes take part
            if (cursor < last && ((uint32_t) __popc(idle) >= a.lines_min_idle || idle == 0xffffffffu)) {
                const uint64_t mine = cursor + __popc(idle & below);
                cursor += __popc(idle);
                if (!busy && mine < last) {
                    line = mine;
                    const uint64_t b = a.offsets[line];
                    const uint64_t e = a.offsets[line + 1] - a.trim;
                    const uint8_t* p = a.corpus + b;
                    const uint32_t len = e > b ? (uint32_t) (e - b) : 0u;
                    mis = (uint32_t) (reinterpret_cast<uintptr_t>(p) & 15);
                    chunk = p - mis;
                    span = mis + len;
                    pieces = len ? (span + 15) >> 4 : 0;
                    piece = 0;
                    SetFull(t, s, a.start);
                    busy = true;
                    if (pieces)
                        cur = LoadChunk16(chunk, buf_lo, buf_hi);
                }
            }
            if (!__any_sync(0xffffffffu, busy))
                break;
            if (busy) {
                // up to kPiecesPerTurn chunks before the lanes look for new lines again: most lines end within
                // one turn, and the bookkeeping around a turn costs as much as walking two chunks
#pragma unroll 1
                for (uint32_t turn = 0; turn < a.lines_turn && piece < pieces; ++turn) {
                    uint4 next = make_uint4(0, 0, 0, 0);
                    if (piece + 1 < pieces)
                        next = LoadChunk16(chunk + 16 * (size_t) (piece + 1), buf_lo, buf_hi);
                    const uint32_t skip = piece == 0 ? mis : 0;
                    const uint32_t left = span - 16 * piece;
                    const uint32_t upto = left < 16 ? left : 16;
                    EdgeFast<kPred>(t, s, skip ? EdgeBytes(cur, skip).Words() : cur, upto - skip);
                    cur = next;
                    ++piece;
                }
                if (piece >= pieces) {
                    ReportScattered(a, t, s, line, true);
                    busy = false;
                }
            }
        }
    }
}

// ---------------------------------------------------------------- lines of text, in stream
//
// The lines of a newline-delimited text lie back to back, so they can be scanned where they are: the text is cut
// into segments of about kTextSegment bytes on 32-byte boundaries of the address space, lane j of a warp walks segment
// 32 * unit + j like the uniform kernel walks a string (32-byte loads, one block ahead in registers, every lane busy in
// every step), and owns the lines that START inside its segment -- it runs past the segment's end until the last of
// them is finished.  What makes this cheap:
//   * the copy of the hot rows in shared memory maps '\n' to the start state in every row (the sink row keeps the
//     sink), so the walk restarts by itself behind a line: no branch, no second pass over the rest of a chunk;
//   * the thirty-two states of a block are packed into eight registers as they appear (one IMAD each, FMA pipe), and
//     the newlines of the block are found in its bytes (exact zero-byte test of word ^ 0x0a0a0a0a, compressed to one
//     bit per byte by a multiply): a lane with newlines parks the packed states in shared memory, picks the state in
//     front of each newline with one LDS.U8 and reports it through a copy of the hot states' reports in shared memory
//     -- the steady state reads no offsets and has no dependent global load;
//   * a lane outside the hot rows at the end of a chunk (the sink is absorbing) replays the chunk byte by byte, line
//     ends included; so does a lane over the unaligned start of its first line.
// The offsets must be those of pire_gpu_split_lines for this text: line i + 1 starts right behind the '\n' of line i.
// They are read once per lane and unit, by the binary search for the first line that starts in the segment; from then
// on line numbers just count up.  Bytes outside the text read as '\n': that ends a last line without newline.
constexpr uint32_t kTextSegment = 4096;
constexpr int kTextBlocksPerSM = 2;
constexpr size_t kTextFinBytes = 256 * sizeof(DeviceFin);
constexpr size_t kTextPackBytes = (size_t) kBlock * 32;     // packed states of one 32-byte block per lane

struct TextLane {
    uint32_t line;       // the line being walked
    int32_t left;        // bytes from the chunk being walked to the end of the segment (negative behind it)
    bool active;         // false: no line of this segment is left
};

// which outputs a line writes: bit 0 accept_masks, bit 1 state_idx, bit 2 match_bits (kept in a register: the
// pointers themselves are 64-bit kernel parameters, and testing them costs three instructions each per line)
__device__ __forceinline__ uint32_t TextOutputs(const ScanArgs& a)
{
    uint32_t outs = (a.accept_masks ? 1u : 0u) | (a.state_idx ? 2u : 0u) | (a.match_bits ? 4u : 0u);
    asm volatile("mov.u32 %0, %0;" : "+r"(outs));
    return outs;
}

__device__ __forceinline__ void TextReport(const ScanArgs& a, uint32_t outs, uint32_t line, DeviceFin f)
{
    if ((outs & 4u) && (f.result >> 31))
        atomicOr(&a.match_bits[line >> 5], 1u << (line & 31));
    if (outs & 1u)
        a.accept_masks[line] = f.mask;
    if (outs & 2u)
        a.state_idx[line] = f.result & 0x7fffffffu;
}

// Bytes [from, to) of the block at text position cpos, one at a time from the complete state `full`.
__device__ __forceinline__ void TextSlow(const ScanArgs& a, const Tables& t, const DeviceFin* fin_hot, uint32_t outs, TextLane& c,
                                         LaneState& s, uint32_t full, int64_t cpos, uint32_t from, uint32_t to, uint64_t seg_hi,
                                         uint64_t total)
{
    for (uint32_t j = from; j < to; ++j) {
        const uint64_t at = (uint64_t) (cpos + (int64_t) j);
        const uint32_t b = at < total ? a.corpus[at] : (uint32_t) '\n';
        if (b == '\n') {
            TextReport(a, outs, c.line, full < t.H ? fin_hot[full] : a.fin[full]);
            ++c.line;
            full = a.start;
            if (c.line >= a.n || at + 1 >= seg_hi) {
                c.active = false;
                break;
            }
            continue;
        }
        full = SlowStep(t, full, b);
    }
    SetFull(t, s, full);
}

// Four steps; q collects the state IN FRONT of each byte (byte 3 - i of q for byte i of w).
template <bool kPred>
__device__ __forceinline__ void TextWord(const Tables& t, uint32_t& g, uint32_t w, uint32_t& q)
{
#pragma unroll
    for (uint32_t i = 0; i < 4; ++i) {
        asm("mad.lo.u32 %0, %0, 256, %1;" : "+r"(q) : "r"(g));       // q = q << 8 | g, on the FMA pipe
        FastStep<kPred>(t, g, w, 0x5540u + i);
    }
}

// Bit i of the result: byte i of w is '\n'.  Exact (no borrow between bytes): 0x80 in every byte of x that is zero,
// then the four flags gathered into the top nibble by one multiply (the partial products do not collide).
__device__ __forceinline__ uint32_t NewlineNibble(uint32_t w)
{
    const uint32_t x = w ^ 0x0a0a0a0au;
    const uint32_t flags = ~(((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x | 0x7f7f7f7fu);
    return (flags * 0x00204081u) >> 28;
}

// One 32-byte block at text position cpos.  `packs` = this lane's slot in the warp's staging area for packed states:
// word w (0..7) of the block's states at packs + (w / 4) * 512 + (w % 4) * 4, so that the two 16-byte stores of a warp
// are contiguous.
template <bool kPred>
__device__ __forceinline__ void TextBlock(const ScanArgs& a, const Tables& t, const DeviceFin* fin_hot, uint32_t outs, TextLane& c,
                                          LaneState& s, uint4 v0, uint4 v1, uint32_t packs, int64_t cpos, uint64_t seg_hi,
                                          uint64_t total)
{
    const uint32_t before = s.g;
    uint32_t g = before;
    uint4 q0 = make_uint4(0, 0, 0, 0), q1 = q0;
    TextWord<kPred>(t, g, v0.x, q0.x);
    TextWord<kPred>(t, g, v0.y, q0.y);
    TextWord<kPred>(t, g, v0.z, q0.z);
    TextWord<kPred>(t, g, v0.w, q0.w);
    TextWord<kPred>(t, g, v1.x, q1.x);
    TextWord<kPred>(t, g, v1.y, q1.y);
    TextWord<kPred>(t, g, v1.z, q1.z);
    TextWord<kPred>(t, g, v1.w, q1.w);
    const int32_t left = c.left;
    c.left = left - 32 > -(1 << 30) ? left - 32 : -(1 << 30);
    if (!c.active)
        return;
    if (g == t.H) {
        // the sink is absorbing (its '\n' entry too): the lane was, or fell, outside the hot rows somewhere in the block
        TextSlow(a, t, fin_hot, outs, c, s, before == t.H ? s.cold : before, cpos, 0, 32, seg_hi, total);
        return;
    }
    s.g = g;
    uint32_t ends = NewlineNibble(v0.x) | (NewlineNibble(v0.y) << 4) | (NewlineNibble(v0.z) << 8) | (NewlineNibble(v0.w) << 12) |
                    (NewlineNibble(v1.x) << 16) | (NewlineNibble(v1.y) << 20) | (NewlineNibble(v1.z) << 24) | (NewlineNibble(v1.w) << 28);
    if (ends == 0)
        return;
    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(packs), "r"(q0.x), "r"(q0.y), "r"(q0.z), "r"(q0.w) : "memory");
    asm volatile("st.shared.v4.u32 [%0+512], {%1,%2,%3,%4};" ::"r"(packs), "r"(q1.x), "r"(q1.y), "r"(q1.z), "r"(q1.w) : "memory");
    const uint32_t n_lines = (uint32_t) a.n;
    do {
        const uint32_t k = (uint32_t) __ffs((int) ends) - 1u;
        ends &= ends - 1u;
        // the state in front of byte k: byte 3 - k % 4 of word k / 4 -- a hot state, the lane is not in the sink
        uint32_t st;
        asm volatile("ld.shared.u8 %0, [%1];" : "=r"(st) : "r"(packs + ((k & 16u) << 5) + ((k & 15u) ^ 3u)) : "memory");
        TextReport(a, outs, c.line, fin_hot[st]);
        ++c.line;
        if (c.line >= n_lines || (int32_t) k + 1 >= left) {         // the next line starts behind the segment
            c.active = false;
            break;
        }
    } while (ends);
}

// A 16-byte chunk that may stick out of the text at either end: bytes outside read as '\n'.  Out of line, it is rare.
__device__ __noinline__ uint4 LoadText16Clipped(const uint8_t* aligned, uintptr_t buf_lo, uintptr_t buf_hi)
{
    uint32_t w[4] = {0x0a0a0a0au, 0x0a0a0a0au, 0x0a0a0a0au, 0x0a0a0a0au};
    for (int k = 0; k < 16; ++k) {
        const uintptr_t at = reinterpret_cast<uintptr_t>(aligned) + k;
        if (at >= buf_lo && at < buf_hi)
            w[k >> 2] = (w[k >> 2] & ~(0xffu << (8 * (k & 3)))) | ((uint32_t) aligned[k] << (8 * (k & 3)));
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

__device__ __forceinline__ void LoadBlock32(const uint8_t* aligned, uintptr_t buf_lo, uintptr_t buf_hi, uint4& v0, uint4& v1)
{
    if (reinterpret_cast<uintptr_t>(aligned) >= buf_lo && reinterpret_cast<uintptr_t>(aligned) + 32 <= buf_hi) {
        LoadStream32(aligned, v0, v1);
    } else {
        v0 = LoadText16Clipped(aligned, buf_lo, buf_hi);
        v1 = LoadText16Clipped(aligned + 16, buf_lo, buf_hi);
    }
}

template <bool kPred>
__global__ void __launch_bounds__(kBlock, kTextBlocksPerSM) ScanTextKernel(const __grid_constant__ ScanArgs a)
{
    uint8_t* const smem = pire_b200_smem;
    SharedView sv = CarveShared(smem, a.hot);
    StageTables(a, sv, a.hot8, a.hot);
    // behind a line the walk starts over: '\n' leads to the start state from every hot row
    for (uint32_t g = threadIdx.x; g < a.hot; g += blockDim.x)
        sv.hot[g * kHotStride + '\n'] = (uint8_t) a.start;
    // what a line that stops in a hot state reports
    DeviceFin* const fin_hot = reinterpret_cast<DeviceFin*>(sv.stage);
    for (uint32_t g = threadIdx.x; g < a.hot; g += blockDim.x)
        fin_hot[g] = a.fin[g];
    __syncthreads();

    Tables t;
    t.hot = sv.hot;
    t.base = SmemAddr(sv.hot);
    t.cls = sv.cls;
    t.full = a.full;
    t.H = a.hot;
    t.letters = a.letters;
    t.wide = a.wide;
    t.m0 = a.exit_bitmap0 | (1u << ('\n' & 31));       // the exit filter must let the separator through

    const uint32_t lane = threadIdx.x & 31;
    const uint32_t outs = TextOutputs(a);
    const uint32_t packs = SmemAddr(sv.stage) + (uint32_t) kTextFinBytes + (threadIdx.x >> 5) * 1024u + lane * 16u;
    const uint64_t total = a.offsets[a.n] - 1;           // position of the last separator (real or the end of the text)
    const uintptr_t buf_lo = reinterpret_cast<uintptr_t>(a.corpus);
    const uintptr_t buf_hi = buf_lo + total;
    const uint32_t mis0 = (uint32_t) (buf_lo & 31);
    const uint64_t warps = (uint64_t) gridDim.x * kWarpsPerBlock;
    // Segment size: about kTextSegment bytes, chosen so that the units (32 segments) come out as a whole number of
    // rounds over the grid's warps -- with a couple of units per warp, one unit more or less is a third of the run time.
    const uint64_t lanes = 32 * warps;
    const uint64_t rounds = (total + 64 + lanes * kTextSegment - 1) / (lanes * kTextSegment);
    uint64_t seg = ((total + 64 + lanes * rounds - 1) / (lanes * rounds) + 31) / 32 * 32;
    seg = seg < 64 ? 64 : seg;
    const uint64_t segments = (total + mis0) / seg + 1;
    const uint64_t units = (segments + 31) / 32;

    for (uint64_t unit = (uint64_t) blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5); unit < units; unit += warps) {
        const uint64_t sidx = unit * 32 + lane;
        const uint64_t seg_hi = (sidx + 1) * seg - mis0;
        TextLane c;
        c.line = 0;
        c.left = 0;
        c.active = false;
        LaneState s;
        s.g = a.start;
        s.cold = 0;
        const uint8_t* p = a.corpus;
        int64_t pos = 0;
        if (sidx < segments) {
            const uint64_t seg_lo = sidx * seg > mis0 ? sidx * seg - mis0 : 0;
            uint64_t lo = 0, hi = a.n;              // first line that starts at or behind seg_lo
            while (lo < hi) {
                const uint64_t mid = (lo + hi) >> 1;
                if (a.offsets[mid] < seg_lo)
                    lo = mid + 1;
                else
                    hi = mid;
            }
            if (lo < a.n) {
                const uint64_t pos0 = a.offsets[lo];
                if (pos0 < seg_hi) {
                    c.line = (uint32_t) lo;
                    c.active = true;
                    pos = (int64_t) ((pos0 + mis0) & ~31ull) - (int64_t) mis0;      // the 32-byte block the line starts in
                    const uint32_t skip = (uint32_t) ((int64_t) pos0 - pos);
                    if (skip) {
                        // the line starts inside the block: the rest of the block byte by byte
                        TextSlow(a, t, fin_hot, outs, c, s, a.start, pos, skip, 32, seg_hi, total);
                        pos += 32;
                    }
                    p = a.corpus + pos;
                    c.left = (int32_t) ((int64_t) seg_hi - pos);
                }
            }
        }
        uint4 v0 = make_uint4(0, 0, 0, 0), v1 = v0;
        if (c.active)
            LoadBlock32(p, buf_lo, buf_hi, v0, v1);
        while (__any_sync(0xffffffffu, c.active)) {
            uint4 n0 = make_uint4(0, 0, 0, 0), n1 = n0;
            if (c.active)
                LoadBlock32(p + 32, buf_lo, buf_hi, n0, n1);
            TextBlock<kPred>(a, t, fin_hot, outs, c, s, v0, v1, packs, pos, seg_hi, total);
            v0 = n0;
            v1 = n1;
            p += 32;
            pos += 32;
        }
    }
}

// ---------------------------------------------------------------- PRIV variant
//
// The plain walk is bound by shared-memory wavefronts once lanes sit in different
// rows (glued scanners: more than two wavefronts per load).  Here the hottest rows
// are replicated into all 32 banks: lane l reads only bank l, so every load is one
// wavefront whatever the states and bytes are.  Layout (byte address inside the
// private region):   [19:14] quad q   [13:7] byte b (< 128)   [6:2] lane   [1:0] row-in-quad s
// A lane's state is its private row id e = 4q + s; one step is
//     e = LDS.U8 [priv + (((e * 0x1001) & 0xFC003) | (b << 7) | (lane << 2))]
// (the multiply drops s into bits 1:0 and q into bits 19:14; the other fields are
// disjoint, so one LOP3 assembles the address).  Rows that are not private map to the
// sink row; a lane found in the sink after a 4-byte word (or a word holding a byte
// >= 128) re-walks that word through the shared hot rows / the complete table and
// re-enters a private row when it can.

constexpr int kPrivBlock = 1024;
constexpr uint32_t kPrivMask = 0x000FC003u;

__device__ __forceinline__ uint32_t LoadSharedU8(uint32_t shared_addr)
{
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(shared_addr));
    return v;
}

// Four steps.  `e` is the lane's private row id.  One step costs two ALU-pipe
// instructions (PRMT, LOP3), three FMA-pipe ones (IMAD x3) and one conflict-free LDS.
// lane_base = shared-window address of the private region + lane * 4.
__device__ __forceinline__ void PrivWord(uint32_t& e, uint32_t w, uint32_t lane_base)
{
    // The private rows cover bytes 0..127 only.  A byte >= 128 sends the whole chunk to the
    // re-walk anyway (PrivChunk), but its speculative step must not index past the table:
    // clear bit 7 of every byte first (one LOP3 per word).
    w &= 0x7F7F7F7Fu;
    const uint32_t k0 = __byte_perm(w, 0, 0x4440) * 128u + lane_base;
    const uint32_t k1 = __byte_perm(w, 0, 0x4441) * 128u + lane_base;
    const uint32_t k2 = __byte_perm(w, 0, 0x4442) * 128u + lane_base;
    const uint32_t k3 = __umulhi(w, 256u) * 128u + lane_base;           // w >> 24 without the ALU pipe
    e = LoadSharedU8(((e * 0x1001u) & kPrivMask) + k0);
    e = LoadSharedU8(((e * 0x1001u) & kPrivMask) + k1);
    e = LoadSharedU8(((e * 0x1001u) & kPrivMask) + k2);
    e = LoadSharedU8(((e * 0x1001u) & kPrivMask) + k3);
}

// Sixteen input bytes.  The sink row is absorbing, so one test per chunk finds every lane
// that left the private rows (or met a byte >= 128, which the private rows do not cover);
// such a lane re-walks the chunk through the shared hot rows (PRMT + LDS per byte, as in the
// plain kernel) and through the complete table only if that fails too.
__device__ __forceinline__ void PrivChunk(const Tables& t, uint32_t& e, uint32_t& other, uint4 v, uint32_t lane_base,
                                          uint32_t sink_id, uint32_t real_rows)
{
    const uint32_t before = e;
    PrivWord(e, v.x, lane_base);
    PrivWord(e, v.y, lane_base);
    PrivWord(e, v.z, lane_base);
    PrivWord(e, v.w, lane_base);
    if (e == sink_id || ((v.x | v.y | v.z | v.w) & 0x80808080u) != 0) {
        const uint32_t from = before == sink_id ? other : before;
        uint32_t g = from < t.H ? from : t.H;
        FastWord<false>(t, g, v.x);
        FastWord<false>(t, g, v.y);
        FastWord<false>(t, g, v.z);
        FastWord<false>(t, g, v.w);
        uint32_t full = g;
        if (g == t.H)
            full = ReplayChunk(t.hot, t.cls, t.full, t.H, t.letters | (t.wide << 31), from, v);
        if (full < real_rows) {
            e = full;
        } else {
            e = sink_id;
            other = full;
        }
    }
}

__global__ void __launch_bounds__(kPrivBlock, 1) ScanUniformPrivKernel(const __grid_constant__ ScanArgs a)
{
    uint8_t* const smem = pire_b200_smem;
    SharedView sv = CarveShared(smem, a.hot_small, a.priv_rows);
    StageTables(a, sv, a.hot8_small, a.hot_small);
    {
        // replicate every packed word into the 32 banks
        const uint32_t words = (a.priv_rows / 4) * 128 * 32;
        uint32_t* dst = reinterpret_cast<uint32_t*>(sv.priv);
        for (uint32_t i = threadIdx.x; i < words; i += blockDim.x)
            dst[i] = __ldg(a.priv_packed + (i >> 5));
        __syncthreads();
    }

    Tables t;
    t.hot = sv.hot;
    t.base = SmemAddr(sv.hot);
    t.cls = sv.cls;
    t.full = a.full;
    t.H = a.hot_small;          // the second tier seen by this kernel
    t.letters = a.letters;
    t.wide = a.wide;
    t.m0 = 0;

    const uint32_t lane = threadIdx.x & 31;
    const uint32_t lane_base = SmemAddr(sv.priv) + (lane << 2);
    const uint32_t real_rows = a.priv_rows - 1 < a.hot_small ? a.priv_rows - 1 : a.hot_small;
    const uint32_t sink_id = a.priv_rows - 1;
    const uint64_t units = (a.n + 31) / 32;
    const uint64_t warps = (uint64_t) gridDim.x * (kPrivBlock / 32);
    const uint32_t len = (uint32_t) a.fixed_len;

    for (uint64_t unit = (uint64_t) blockIdx.x * (kPrivBlock / 32) + (threadIdx.x >> 5); unit < units; unit += warps) {
        const uint64_t i = unit * 32 + lane;
        const bool valid = i < a.n;
        const uint8_t* p = a.corpus + (valid ? i : a.n - 1) * (uint64_t) len;

        uint32_t other = a.start;
        uint32_t e = a.start < real_rows ? a.start : sink_id;

        uint4 c0, c1, d0, d1;
        LoadStream32(p, c0, c1);
        for (uint32_t off = 0;;) {
            off += 32;
            const bool more_d = off < len;
            if (more_d)
                LoadStream32(p + off, d0, d1);
            PrivChunk(t, e, other, c0, lane_base, sink_id, real_rows);
            PrivChunk(t, e, other, c1, lane_base, sink_id, real_rows);
            if (!more_d)
                break;
            off += 32;
            const bool more_c = off < len;
            if (more_c)
                LoadStream32(p + off, c0, c1);
            PrivChunk(t, e, other, d0, lane_base, sink_id, real_rows);
            PrivChunk(t, e, other, d1, lane_base, sink_id, real_rows);
            if (!more_c)
                break;
        }

        LaneState fs;
        fs.g = t.H;
        fs.cold = e == sink_id ? other : e;
        Report(a, t, fs, unit, i, valid);
    }
}

__device__ __forceinline__ uint32_t FullNext(const Tables& t, uint32_t s, uint32_t letter)
{
    size_t at = (size_t) s * t.letters + letter;
    return t.wide ? __ldg(static_cast<const uint32_t*>(t.full) + at) : (uint32_t) __ldg(static_cast<const uint16_t*>(t.full) + at);
}

// ---------------------------------------------------------------- prefix and suffix scans
//
// Pire::LongestPrefix / ShortestPrefix (run.h:277-311, predicates run.h:69-100) and LongestSuffix /
// ShortestSuffix (run.h:316-362) for a batch: the same walk, but Final() and Dead() matter after every
// byte -- the longest scan remembers the last position whose state is final, the shortest stops at the
// first, both stop in a dead state (pire_ut.cpp ScanTermination@475).  The suffix scans walk the string
// from its last byte to its first (the scanner is normally built from Fsm::Reverse()).  One string per
// lane through the generic kernel's machinery (cp.async ring, fused hot rows).  Final hot states carry the
// highest hot ids, so the maximum id over the 16 steps of a chunk says whether the chunk entered a final
// state or left the hot rows; such a chunk is walked again, branch-free, marking where; only a chunk that
// leaves the hot rows is replayed byte by byte with the predicate.  A dead state is never final and only
// leads to dead states, so noticing it late cannot change the answer: it is looked for once per ring round
// (64 bytes) to stop the lane, and a lane that has stopped no longer fetches its string.
struct PrefixLane {
    uint32_t consumed;      // bytes walked so far
    uint32_t pos;           // answer so far, kNoPrefix = none
    bool stop;
    static constexpr bool kAnyFinal = true;     // every final state counts (not one regexp's)
};
constexpr uint32_t kNoPrefix = 0xFFFFFFFFu;

// The bytes of an edge chunk from index `top` downwards (suffix scans).
struct EdgeBytesDown {
    uint64_t lo, hi;
    __device__ __forceinline__ EdgeBytesDown(uint4 v, uint32_t top)
    {
        lo = (uint64_t) v.x | ((uint64_t) v.y << 32);
        hi = (uint64_t) v.z | ((uint64_t) v.w << 32);
        uint32_t drop = 15 - top;                       // bytes above `top` are not ours
        if (drop >= 8) {
            hi = lo;
            lo = 0;
            drop -= 8;
        }
        if (drop) {
            hi = (hi << (8 * drop)) | (lo >> (64 - 8 * drop));
            lo <<= 8 * drop;
        }
    }
    __device__ __forceinline__ uint32_t Next()
    {
        uint32_t b = (uint32_t) (hi >> 56);
        hi = (hi << 8) | (lo >> 56);
        lo <<= 8;
        return b;
    }
};

template <bool kShortest>
__device__ __forceinline__ void PrefixCheck(const ScanArgs& a, uint32_t H, const uint8_t* hot_flags, uint32_t state, PrefixLane& l)
{
    const uint32_t fl = state < H ? hot_flags[state] : __ldg(a.flags + state);
    if (fl & 1u) {                                                   // Final: run.h:76-79 / :92-93 / :329-330 / :353
        l.pos = l.consumed;
        l.stop = kShortest;
    }
    if (fl & 2u)                                                     // Dead: run.h:82 / :94 / :328 / :353
        l.stop = true;
}

// Whether hot id h (or H) counts in the branch-free replay of PrefixChunk16.
__device__ __forceinline__ bool HotAccepts(const ScanArgs& a, uint32_t h, const PrefixLane&) { return h >= a.first_final_hot; }

template <bool kShortest, bool kReverse, class Lane = PrefixLane>
__device__ __forceinline__ void PrefixChunk16(const ScanArgs& a, const Tables& t, const uint8_t* hot_flags, LaneState& s, uint4 v,
                                              Lane& l)
{
    const uint32_t before = s.g;
    uint32_t g = before, top = 0, low = 0xffffffffu;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
        const int at = kReverse ? 3 - w : w;
        const uint32_t word = at == 0 ? v.x : at == 1 ? v.y : at == 2 ? v.z : v.w;
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            FastStep<false, false>(t, g, word, 0x5540 + (kReverse ? 3 - b : b));
            top = max(top, g);
            if (!kShortest)
                low = min(low, g);
        }
    }
    if (top < a.first_final_hot) {           // sixteen steps through non-final hot states
        s.g = g;
        l.consumed += 16;
        return;
    }
    if (!kShortest && Lane::kAnyFinal && low >= a.first_final_hot && top != t.H) {
        // sixteen steps through final hot states (a lane behind an unanchored match sits in such states for the rest of
        // its string): the longest prefix so far ends with this chunk, no second pass needed
        s.g = g;
        l.consumed += 16;
        l.pos = l.consumed;
        return;
    }
    // ShortestSuffix steps BeginMark from the state it stopped in (run.h:357-359), so that scan needs the
    // state at the first final step, not the one after the chunk: it goes straight to the byte-wise replay
    // (once per string).
    if (before != t.H && !(kShortest && kReverse)) {
        // a final state (or the sink) was entered: the chunk again, branch-free, noting where.  `mark` is the
        // 1-based step of the last (longest) or first (shortest) final state entered; the sink id also
        // compares >= first_final_hot, but a lane that reached the sink takes the slow path below instead.
        uint32_t h = before, mark = 0;
#pragma unroll
        for (int w = 0; w < 4; ++w) {
            const int at = kReverse ? 3 - w : w;
            const uint32_t word = at == 0 ? v.x : at == 1 ? v.y : at == 2 ? v.z : v.w;
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                FastStep<false, false>(t, h, word, 0x5540 + (kReverse ? 3 - b : b));
                const bool final = HotAccepts(a, h, l);
                if (kShortest)
                    mark = final && mark == 0 ? (uint32_t) (4 * w + b + 1) : mark;
                else
                    mark = final ? (uint32_t) (4 * w + b + 1) : mark;
            }
        }
        if (h != t.H) {
            if (mark) {
                l.pos = l.consumed + mark;
                l.stop = kShortest;
            }
            l.consumed += 16;
            s.g = h;
            return;
        }
    }
    uint32_t full = before == t.H ? s.cold : before;
    if (kReverse) {
        EdgeBytesDown eb(v, 15);
        for (int k = 0; k < 16 && !l.stop; ++k) {
            full = SlowStep(t, full, eb.Next());
            ++l.consumed;
            PrefixCheck<kShortest>(a, t.H, hot_flags, full, l);
        }
    } else {
        EdgeBytes eb(v, 0);
        for (int k = 0; k < 16 && !l.stop; ++k) {
            full = SlowStep(t, full, eb.Next());
            ++l.consumed;
            PrefixCheck<kShortest>(a, t.H, hot_flags, full, l);
        }
    }
    SetFull(t, s, full);
}

template <bool kShortest, bool kReverse>
__global__ void __launch_bounds__(kBlock, kGenericBlocksPerSM) PrefixKernel(const __grid_constant__ ScanArgs a)
{
    uint8_t* const smem = pire_b200_smem;
    SharedView sv = CarveShared(smem, a.hot);
    StageTables(a, sv, a.hot8, a.hot);
    uint8_t* const hot_flags = sv.stage + kStageBytes;              // H + 1 bytes behind the staging ring
    for (uint32_t i = threadIdx.x; i <= a.hot; i += blockDim.x)
        hot_flags[i] = i < a.hot ? a.flags[i] : 0;
    __syncthreads();

    Tables t;
    t.hot = sv.hot;
    t.base = SmemAddr(sv.hot);
    t.cls = sv.cls;
    t.full = a.full;
    t.H = a.hot;
    t.letters = a.letters;
    t.wide = a.wide;
    t.m0 = 0;

    const uint32_t lane = threadIdx.x & 31;
    const uint64_t units = (a.n + 31) / 32;
    const uint64_t warps = (uint64_t) gridDim.x * kWarpsPerBlock;
    const uint32_t stage = SmemAddr(sv.stage) + (((threadIdx.x >> 5) * kStageSlots) * 32 + lane) * 16;
    const uintptr_t buf_lo = reinterpret_cast<uintptr_t>(a.corpus);
    const uintptr_t buf_hi = buf_lo + (a.offsets ? a.offsets[a.n] - a.trim : a.n * a.fixed_len);

    for (uint64_t unit = (uint64_t) blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5); unit < units; unit += warps) {
        const uint64_t i = unit * 32 + lane;
        const bool valid = i < a.n;
        uint64_t b = 0, e = 0;
        if (valid) {
            if (a.offsets) {
                b = a.offsets[i];
                e = a.offsets[i + 1] - a.trim;
                e = e < b ? b : e;       // an empty entry of a trimmed (lines) batch, or caller offsets that step back
            } else {
                b = i * a.fixed_len;
                e = b + a.fixed_len;
            }
        }
        const uint8_t* const first = a.corpus + b;
        const uint8_t* const end = a.corpus + e;
        const uint32_t len = (uint32_t) (e - b);

        // Initialize() and the first mark: BeginMark for a prefix scan (run.h:282-283), EndMark for a
        // suffix scan (run.h:321-322)
        uint32_t full = a.initial;
        if (a.with_begin)
            full = FullNext(t, full, a.begin_class);
        PrefixLane l;
        l.consumed = 0;
        l.pos = kNoPrefix;
        l.stop = !valid;
        {
            const uint32_t fl = full < t.H ? hot_flags[full] : __ldg(a.flags + full);
            if (fl & 1u) {                                               // run.h:284 / :301-302 / :329-330 / :353
                l.pos = 0;
                l.stop = l.stop || kShortest;
            }
            if (kReverse && (fl & 2u))                                   // run.h:328 / :353: Dead is looked at before the first byte
                l.stop = true;
        }
        // edge bytes on the side the walk starts from, up to a 16-byte boundary
        const uint8_t* p = kReverse ? end : first;                       // forward: next byte; reverse: one past the next byte
        {
            const uint32_t misalign = (uint32_t) (reinterpret_cast<uintptr_t>(p) & 15);
            if (len != 0 && misalign != 0) {
                const uint32_t span = kReverse ? misalign : 16 - misalign;      // bytes between p and the boundary
                const uint32_t nedge = len < span ? len : span;
                const uint8_t* chunk = p - misalign;
                if (!l.stop) {
                    const bool whole = reinterpret_cast<uintptr_t>(chunk) >= buf_lo && reinterpret_cast<uintptr_t>(chunk) + 16 <= buf_hi;
                    if (kReverse) {
                        EdgeBytesDown eb(whole ? LoadEdge16(chunk) : make_uint4(0, 0, 0, 0), misalign - 1);
                        for (uint32_t k = 0; k < nedge && !l.stop; ++k) {
                            const uint32_t byte = whole ? eb.Next() : (uint32_t) p[-1 - (int) k];
                            full = SlowStep(t, full, byte);
                            ++l.consumed;
                            PrefixCheck<kShortest>(a, t.H, hot_flags, full, l);
                        }
                    } else {
                        EdgeBytes eb(whole ? LoadEdge16(chunk) : make_uint4(0, 0, 0, 0), misalign);
                        for (uint32_t k = 0; k < nedge && !l.stop; ++k) {
                            const uint32_t byte = whole ? eb.Next() : (uint32_t) p[k];
                            full = SlowStep(t, full, byte);
                            ++l.consumed;
                            PrefixCheck<kShortest>(a, t.H, hot_flags, full, l);
                        }
                    }
                }
                p = kReverse ? p - nedge : p + nedge;
            }
        }
        LaneState s;
        SetFull(t, s, full);
        if (!kReverse && a.uniform) {
            // Fixed-length, 32-byte aligned batch (the BASELINE configs' shape): no edge bytes, and the strings stream
            // through registers like in the uniform scan kernel -- one pair of LDG.128 per lane per 32 bytes, prefetched one
            // block ahead -- instead of the cp.async ring, whose shared-memory round trip costs half a wavefront per
            // step on the pipe that bounds the walk.
            // every lane of the warp walks the loop (its control flow holds a warp vote), also the lanes past the end
            // of the batch: they are stopped from the start and read string 0
            const uint32_t ulen = (uint32_t) a.fixed_len;
            const uint8_t* const src = valid ? first : a.corpus;
            if (ulen != 0) {
                uint4 a0, a1, b0, b1;
                LoadStream32(src, a0, a1);
                for (uint32_t off = 0;;) {
                    off += 32;
                    const bool more_b = off < ulen;
                    if (more_b)
                        LoadStream32(src + off, b0, b1);
                    if (!l.stop)
                        PrefixChunk16<kShortest, kReverse>(a, t, hot_flags, s, a0, l);
                    if (!l.stop)
                        PrefixChunk16<kShortest, kReverse>(a, t, hot_flags, s, a1, l);
                    if (!more_b)
                        break;
                    off += 32;
                    const bool more_a = off < ulen;
                    if (more_a)
                        LoadStream32(src + off, a0, a1);
                    if (!l.stop)
                        PrefixChunk16<kShortest, kReverse>(a, t, hot_flags, s, b0, l);
                    if (!l.stop)
                        PrefixChunk16<kShortest, kReverse>(a, t, hot_flags, s, b1, l);
                    // a dead state only leads to dead states: stop the lane once it is noticed (every 64 bytes)
                    if (!l.stop) {
                        const uint32_t at = FullState(t, s);
                        if ((at < t.H ? hot_flags[at] : __ldg(a.flags + at)) & 2u)
                            l.stop = true;
                    }
                    if (!more_a || __all_sync(0xffffffffu, l.stop))
                        break;
                }
            }
            p = end;
        }
        // body: whole 16-byte chunks; chunk c is at p + 16c (forward) or p - 16(c+1) (reverse)
        const uint32_t chunks = (uint32_t) ((kReverse ? p - first : end - p) >> 4);
#pragma unroll
        for (int j = 0; j < kStageSlots; ++j) {
            if ((uint32_t) j < chunks && !l.stop)
                CopyAsync16(stage + j * 512, kReverse ? p - 16 * (j + 1) : p + 16 * j);
            CopyAsyncCommit();
        }
        for (uint32_t k = 0; __any_sync(0xffffffffu, k < chunks && !l.stop); k += kStageSlots) {
#pragma unroll
            for (int j = 0; j < kStageSlots; ++j) {
                CopyAsyncWait<kStageSlots - 1>();
                const uint4 v = LoadShared16(stage + j * 512);
                const bool had = k + j < chunks && !l.stop;              // this slot was filled for this lane
                if (k + kStageSlots + j < chunks && !l.stop) {
                    const size_t c = (size_t) k + kStageSlots + j;
                    CopyAsync16(stage + j * 512, kReverse ? p - 16 * (c + 1) : p + 16 * c);
                }
                CopyAsyncCommit();
                if (had)
                    PrefixChunk16<kShortest, kReverse>(a, t, hot_flags, s, v, l);
            }
            // a dead state only leads to dead states: stop the lane (and its fetches) once it is noticed
            if (!l.stop) {
                const uint32_t at = FullState(t, s);
                if ((at < t.H ? hot_flags[at] : __ldg(a.flags + at)) & 2u)
                    l.stop = true;
            }
        }
        CopyAsyncWait<0>();
        full = FullState(t, s);
        p = kReverse ? p - 16 * (size_t) chunks : p + 16 * (size_t) chunks;
        // edge bytes on the far side: fewer than 16, p is on a 16-byte boundary
        const uint32_t nfar = (uint32_t) (kReverse ? p - first : end - p);
        if (nfar != 0 && !l.stop) {
            const uint8_t* chunk = kReverse ? p - 16 : p;
            const bool whole = reinterpret_cast<uintptr_t>(chunk) >= buf_lo && reinterpret_cast<uintptr_t>(chunk) + 16 <= buf_hi;
            if (kReverse) {
                EdgeBytesDown eb(whole ? LoadEdge16(chunk) : make_uint4(0, 0, 0, 0), 15);
                for (uint32_t k = 0; k < nfar && !l.stop; ++k) {
                    const uint32_t byte = whole ? eb.Next() : (uint32_t) p[-1 - (int) k];
                    full = SlowStep(t, full, byte);
                    ++l.consumed;
                    PrefixCheck<kShortest>(a, t.H, hot_flags, full, l);
                }
            } else {
                EdgeBytes eb(whole ? LoadEdge16(chunk) : make_uint4(0, 0, 0, 0), 0);
                for (uint32_t k = 0; k < nfar && !l.stop; ++k) {
                    const uint32_t byte = whole ? eb.Next() : (uint32_t) p[k];
                    full = SlowStep(t, full, byte);
                    ++l.consumed;
                    PrefixCheck<kShortest>(a, t.H, hot_flags, full, l);
                }
            }
        }
        if (valid) {
            if (kReverse && kShortest) {
                // run.h:357-360: the last mark is stepped from wherever the scan stopped, and the answer is
                // the stopping place if that state is final
                if (a.through_end)
                    full = FullNext(t, full, a.end_class);
                l.pos = (__ldg(a.flags + full) & 1u) ? l.consumed : kNoPrefix;
            } else if (a.through_end) {                                  // run.h:286-290 / :305-309 / :336-340
                const uint32_t last = FullNext(t, full, a.end_class);
                if ((__ldg(a.flags + last) & 1u) && (!kShortest || l.pos == kNoPrefix))
                    l.pos = len;
            }
            a.prefix_len[i] = l.pos;
        }
    }
}

// Forward prefix scans of a fixed-length, 32-byte aligned batch (the BASELINE configs' shape) in a kernel of their own:
// no edge bytes and no staging ring, so two CTAs of twenty warps fit an SM instead of the generic kernel's two of
// sixteen.  The walk is plain: with the exit filter of hot id 0 its step is five ALU-pipe instructions (PRMT, SHF,
// 2 x LOP3, VIMNMX), about twice the plain step's.  (The look-ahead filter does not carry over at all: it skips the
// one-step states behind an exit byte, and a prefix scan must see them if they are final.)
template <bool kShortest>
__global__ void __maxnreg__(48) PrefixUniformKernel(const __grid_constant__ ScanArgs a)
{
    uint8_t* const smem = pire_b200_smem;
    SharedView sv = CarveShared(smem, a.hot);
    StageTables(a, sv, a.hot8, a.hot);
    uint8_t* const hot_flags = sv.stage;                            // H + 1 bytes, where the generic kernels keep their ring
    for (uint32_t i = threadIdx.x; i <= a.hot; i += blockDim.x)
        hot_flags[i] = i < a.hot ? a.flags[i] : 0;
    __syncthreads();

    Tables t;
    t.hot = sv.hot;
    t.base = SmemAddr(sv.hot);
    t.cls = sv.cls;
    t.full = a.full;
    t.H = a.hot;
    t.letters = a.letters;
    t.wide = a.wide;

    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warps_per_block = blockDim.x >> 5;
    const uint64_t units = (a.n + 31) / 32;
    const uint64_t warps = (uint64_t) gridDim.x * warps_per_block;
    const uint32_t ulen = (uint32_t) a.fixed_len;

    for (uint64_t unit = (uint64_t) blockIdx.x * warps_per_block + (threadIdx.x >> 5); unit < units; unit += warps) {
        const uint64_t i = unit * 32 + lane;
        const bool valid = i < a.n;
        // Initialize() and BeginMark (run.h:282-283)
        uint32_t full = a.initial;
        if (a.with_begin)
            full = FullNext(t, full, a.begin_class);
        PrefixLane l;
        l.consumed = 0;
        l.pos = kNoPrefix;
        l.stop = !valid;
        if ((full < t.H ? hot_flags[full] : __ldg(a.flags + full)) & 1u) {      // run.h:284 / :301-302
            l.pos = 0;
            l.stop = l.stop || kShortest;
        }
        LaneState s;
        SetFull(t, s, full);
        // every lane of the warp walks the loop (its control flow holds a warp vote), also the lanes past the end of
        // the batch: they are stopped from the start and read string 0
        const uint8_t* const src = a.corpus + (valid ? i : 0) * (uint64_t) ulen;
        if (ulen != 0) {
            uint4 a0, a1, b0, b1;
            LoadStream32(src, a0, a1);
            for (uint32_t off = 0;;) {
                off += 32;
                const bool more_b = off < ulen;
                if (more_b)
                    LoadStream32(src + off, b0, b1);
                if (!l.stop)
                    PrefixChunk16<kShortest, false>(a, t, hot_flags, s, a0, l);
                if (!l.stop)
                    PrefixChunk16<kShortest, false>(a, t, hot_flags, s, a1, l);
                if (!more_b)
                    break;
                off += 32;
                const bool more_a = off < ulen;
                if (more_a)
                    LoadStream32(src + off, a0, a1);
                if (!l.stop)
                    PrefixChunk16<kShortest, false>(a, t, hot_flags, s, b0, l);
                if (!l.stop)
                    PrefixChunk16<kShortest, false>(a, t, hot_flags, s, b1, l);
                // a dead state only leads to dead states: stop the lane once it is noticed (every 64 bytes)
                if (!l.stop) {
                    const uint32_t at = FullState(t, s);
                    if ((at < t.H ? hot_flags[at] : __ldg(a.flags + at)) & 2u)
                        l.stop = true;
                }
                if (!more_a || __all_sync(0xffffffffu, l.stop))
                    break;
            }
        }
        if (valid) {
            if (a.through_end) {                                             // run.h:286-290 / :305-309
                const uint32_t last = FullNext(t, FullState(t, s), a.end_class);
                if ((__ldg(a.flags + last) & 1u) && (!kShortest || l.pos == kNoPrefix))
                    l.pos = ulen;
            }
            a.prefix_len[i] = l.pos;
        }
    }
}

// ---------------------------------------------------------------- where the matches start
//
// The leftmost start of a match that ends at a given position (pire_gpu_match_starts_*): Pire::LongestSuffix
// (run.h:316-342) through a scanner built with Fsm::Reverse(), walked from the entry's end leftwards, one entry per lane.
// The walk is the suffix scan's (PrefixChunk16 over 16-byte chunks of a per-lane cp.async ring, edge bytes byte by
// byte); what differs is the lane: positions are 64-bit, "accepted" means the entry's regexp is in the state's accept
// list (the bit of the hot state's mask for ids < 32, the list itself above), and the lane stops as soon as its state can
// no longer reach a state accepting that regexp (ScanTables::live) -- on Dead() alone, a glued reversed scanner would
// keep every entry walking as long as its longest-living sibling regexp.  Noticing that late changes nothing (such a
// state only leads to such states), so it is looked at once per ring round.  Entries come in text order, so the lanes
// of a warp read overlapping bytes; warps of a persistent grid take groups of 32 consecutive entries from a counter, so
// that a few long walks hold up one warp and not a whole CTA's share.
constexpr uint32_t kAnyRegexp = 0xFFFFFFFFu;
constexpr uint64_t kNoStart = ~0ull;
constexpr uint32_t kStartsHotLiveWords = 16;       // live rows up to this many words are staged in shared memory

struct StartsLane {
    uint64_t consumed;          // bytes walked so far
    uint64_t pos;               // longest accepted suffix so far, kNoStart = none
    bool stop;
    uint32_t id;                // the entry's regexp, kAnyRegexp = Final()
    const uint32_t* hot_mask;   // shared, H + 1 words: accept mask (ids < 32) of each final hot state, 0 for the rest
    const uint32_t* hot_live;   // shared: the hot states' rows of ScanArgs::live, or null (read from global memory)
    static constexpr bool kAnyFinal = false;
};

__device__ __forceinline__ bool AcceptsId(const ScanArgs& a, uint32_t state, uint32_t id)
{
    for (uint32_t k = __ldg(a.acc_begin + state), e = __ldg(a.acc_begin + state + 1); k < e; ++k)
        if (__ldg(a.acc_ids + k) == id)
            return true;
    return false;
}

__device__ __forceinline__ bool HotAccepts(const ScanArgs& a, uint32_t h, const StartsLane& l)
{
    if (h < a.first_final_hot || h >= a.hot)
        return false;
    if (l.id < 32 || l.id == kAnyRegexp)
        return l.id == kAnyRegexp || ((l.hot_mask[h] >> l.id) & 1u);
    return AcceptsId(a, h, l.id);
}

// id_k in AcceptedRegexps(state) (Final(state) without an id)
__device__ __forceinline__ bool StartsAccepts(const ScanArgs& a, uint32_t H, const uint8_t* hot_flags, uint32_t state,
                                              const StartsLane& l)
{
    const uint32_t fl = state < H ? hot_flags[state] : __ldg(a.flags + state);
    if (!(fl & 1u))
        return false;
    if (l.id == kAnyRegexp)
        return true;
    if (l.id < 32)
        return ((state < H ? l.hot_mask[state] : __ldg(&a.fin[state].mask)) >> l.id) & 1u;
    return AcceptsId(a, state, l.id);
}

// id_k can still be accepted from `state` (not Dead() without an id)
__device__ __forceinline__ bool StartsLive(const ScanArgs& a, uint32_t H, const uint8_t* hot_flags, uint32_t state,
                                           const StartsLane& l)
{
    if (l.id == kAnyRegexp)
        return !((state < H ? hot_flags[state] : __ldg(a.flags + state)) & 2u);
    const size_t at = (size_t) state * a.live_words + l.id / 32;
    return ((state < H && l.hot_live ? l.hot_live[at] : __ldg(a.live + at)) >> (l.id % 32)) & 1u;
}

template <bool kShortest>
__device__ __forceinline__ void PrefixCheck(const ScanArgs& a, uint32_t H, const uint8_t* hot_flags, uint32_t state, StartsLane& l)
{
    if (StartsAccepts(a, H, hot_flags, state, l))
        l.pos = l.consumed;
    if (!StartsLive(a, H, hot_flags, state, l))
        l.stop = true;
}

__global__ void __launch_bounds__(kBlock, kGenericBlocksPerSM) MatchStartsKernel(const __grid_constant__ ScanArgs a)
{
    uint8_t* const smem = pire_b200_smem;
    SharedView sv = CarveShared(smem, a.hot);
    StageTables(a, sv, a.hot8, a.hot);
    uint8_t* const hot_flags = sv.stage + kStageBytes;                       // H + 1 bytes behind the staging ring
    uint32_t* const hot_mask = reinterpret_cast<uint32_t*>(hot_flags + 272); // H + 1 words
    uint32_t* const hot_live = a.live_words <= kStartsHotLiveWords ? hot_mask + 256 : nullptr;
    for (uint32_t i = threadIdx.x; i <= a.hot; i += blockDim.x) {
        const uint32_t fl = i < a.hot ? a.flags[i] : 0;
        hot_flags[i] = fl;
        hot_mask[i] = (fl & 1u) ? a.fin[i].mask : 0;
    }
    if (hot_live)
        for (uint32_t i = threadIdx.x; i < a.hot * a.live_words; i += blockDim.x)
            hot_live[i] = a.live[i];
    __syncthreads();

    Tables t;
    t.hot = sv.hot;
    t.base = SmemAddr(sv.hot);
    t.cls = sv.cls;
    t.full = a.full;
    t.H = a.hot;
    t.letters = a.letters;
    t.wide = a.wide;
    t.m0 = 0;

    const uint32_t lane = threadIdx.x & 31;
    const uint32_t stage = SmemAddr(sv.stage) + (((threadIdx.x >> 5) * kStageSlots) * 32 + lane) * 16;
    const uintptr_t buf_lo = reinterpret_cast<uintptr_t>(a.corpus);
    const uintptr_t buf_hi = buf_lo + (a.offsets ? a.offsets[a.n] : a.n * a.fixed_len);
    const uint64_t first = a.entries_first ? *a.entries_first : 0;
    const uint64_t found = *a.entries_found;
    const uint64_t last = found < a.ends_capacity ? found : a.ends_capacity;
    if (first >= last)
        return;

    for (;;) {
        unsigned long long group = 0;
        if (lane == 0)
            group = atomicAdd(a.group_counter, 1ull);
        group = __shfl_sync(0xffffffffu, group, 0);
        if (group * 32 >= last - first)
            break;
        const uint64_t k = first + group * 32 + lane;
        bool valid = k < last;
        uint64_t end = 0, wstart = 0, wend = 0;
        const uint8_t* wbase = a.corpus;
        uint32_t id = kAnyRegexp;
        if (valid) {
            const uint32_t si = a.entry_strings ? a.entry_strings[k] : 0;
            end = a.entry_ends[k];
            valid = si < a.n;
            if (valid) {
                uint64_t b, e;
                if (a.offsets) {
                    b = a.offsets[si];
                    e = a.offsets[si + 1];
                    e = e < b ? b : e;
                } else {
                    b = (uint64_t) si * a.fixed_len;
                    e = b + a.fixed_len;
                }
                wend = a.window_end ? a.window_end[si] : a.ends_base + (e - b);
                wstart = wend - (e - b);
                valid = wend >= e - b && end >= wstart && end <= wend;    // entries outside the window are not ours
                wbase = a.corpus + b;
                if (a.entry_ids)
                    id = a.entry_ids[k];
            }
        }
        const uint64_t lower = valid && a.max_back && end - wstart > a.max_back ? end - a.max_back : wstart;
        const bool begin_here = a.with_begin && lower == wstart;
        // an entry at the window's end under END: its match may have taken the EndMark step or not, the longer wins
        const int passes = !valid ? 0 : (a.with_end && end == wend) ? 2 : 1;
        uint64_t best = kNoStart;
        bool open = false;
        for (int pass = 0; __any_sync(0xffffffffu, pass < passes); ++pass) {
            StartsLane l;
            l.consumed = 0;
            l.pos = kNoStart;
            l.stop = pass >= passes;
            l.id = id;
            l.hot_mask = hot_mask;
            l.hot_live = hot_live;
            uint32_t full = pass == 1 ? FullNext(t, a.initial, a.end_class) : a.initial;
            if (!l.stop)
                PrefixCheck<false>(a, t.H, hot_flags, full, l);
            const uint8_t* const lo = wbase + (lower - wstart);
            const uint8_t* p = l.stop ? lo : wbase + (end - wstart);         // one past the next byte
            // edge bytes up to a 16-byte boundary
            {
                const uint32_t misalign = (uint32_t) (reinterpret_cast<uintptr_t>(p) & 15);
                const uint64_t len = (uint64_t) (p - lo);
                if (len != 0 && misalign != 0) {
                    const uint32_t nedge = len < misalign ? (uint32_t) len : misalign;
                    const uint8_t* chunk = p - misalign;
                    const bool whole = reinterpret_cast<uintptr_t>(chunk) >= buf_lo && reinterpret_cast<uintptr_t>(chunk) + 16 <= buf_hi;
                    EdgeBytesDown eb(whole ? LoadEdge16(chunk) : make_uint4(0, 0, 0, 0), misalign - 1);
                    for (uint32_t j = 0; j < nedge && !l.stop; ++j) {
                        full = SlowStep(t, full, whole ? eb.Next() : (uint32_t) p[-1 - (int) j]);
                        ++l.consumed;
                        PrefixCheck<false>(a, t.H, hot_flags, full, l);
                    }
                    p -= nedge;
                }
            }
            LaneState s;
            SetFull(t, s, full);
            // body: whole 16-byte chunks, chunk c at p - 16(c+1)
            const uint64_t chunks = l.stop ? 0 : (uint64_t) (p - lo) >> 4;
#pragma unroll
            for (int j = 0; j < kStageSlots; ++j) {
                if ((uint64_t) j < chunks)
                    CopyAsync16(stage + j * 512, p - 16 * (j + 1));
                CopyAsyncCommit();
            }
            for (uint64_t c = 0; __any_sync(0xffffffffu, c < chunks && !l.stop); c += kStageSlots) {
#pragma unroll
                for (int j = 0; j < kStageSlots; ++j) {
                    CopyAsyncWait<kStageSlots - 1>();
                    const uint4 v = LoadShared16(stage + j * 512);
                    const bool had = c + j < chunks && !l.stop;
                    if (c + kStageSlots + j < chunks && !l.stop)
                        CopyAsync16(stage + j * 512, p - 16 * (c + kStageSlots + j + 1));
                    CopyAsyncCommit();
                    if (had)
                        PrefixChunk16<false, true>(a, t, hot_flags, s, v, l);
                }
                if (!l.stop && !StartsLive(a, t.H, hot_flags, FullState(t, s), l))
                    l.stop = true;
            }
            CopyAsyncWait<0>();
            full = FullState(t, s);
            // edge bytes on the far side: fewer than 16, p - 16 * chunks is on a 16-byte boundary
            if (!l.stop) {
                p -= 16 * chunks;
                const uint32_t nfar = (uint32_t) (p - lo);
                if (nfar != 0) {
                    const uint8_t* chunk = p - 16;
                    const bool whole = reinterpret_cast<uintptr_t>(chunk) >= buf_lo && reinterpret_cast<uintptr_t>(chunk) + 16 <= buf_hi;
                    EdgeBytesDown eb(whole ? LoadEdge16(chunk) : make_uint4(0, 0, 0, 0), 15);
                    for (uint32_t j = 0; j < nfar && !l.stop; ++j) {
                        full = SlowStep(t, full, whole ? eb.Next() : (uint32_t) p[-1 - (int) j]);
                        ++l.consumed;
                        PrefixCheck<false>(a, t.H, hot_flags, full, l);
                    }
                }
            }
            if (pass < passes) {
                // a lane that has not stopped walked every byte down to `lower`
                if (!l.stop) {
                    if (begin_here) {
                        if (StartsAccepts(a, t.H, hot_flags, FullNext(t, full, a.begin_class), l))   // run.h:336-340
                            l.pos = l.consumed;
                    } else if (StartsLive(a, t.H, hot_flags, full, l)) {
                        open = true;
                    }
                }
                if (l.pos != kNoStart && (best == kNoStart || l.pos > best))
                    best = l.pos;
            }
        }
        if (valid) {
            a.match_starts[k] = best == kNoStart ? kNoStart : end - best;
            if (a.match_open)
                a.match_open[k] = open ? 1 : 0;
        }
    }
}

// ---------------------------------------------------------------- counting (HalfFinalScanner)
//
// pire/scanners/half_final.h: the same table walk, but after Initialize() and after every symbol
// TakeAction (:154-163) adds one to the counter of each regexp listed for the state when the state is
// final.  The per-string result is the vector of counters (State::Result, :88-90).
//
// The walk is the generic kernel's (one string per lane, 16-byte chunks through the cp.async ring, fused
// hot rows in shared memory).  Two ways to keep the counters, chosen per automaton on the host:
//  * packed (kWords = 1 or 2, up to 16 regexps): every state has its increments as 8-bit fields of one
//    or two 64-bit words (zero for non-final states; the hot states' words sit in shared memory), so
//    TakeAction is an unconditional 64-bit add per word.  Fields are widened to 16 bits after every
//    chunk and written to the string's row of counters every 120 chunks, before they can wrap;
//  * lists (kWords = 0): the accept list of a final state is walked; counters 0..3 in registers, the
//    rest straight in the string's row in global memory (lane-private, no atomics).
// Final hot states carry the highest hot ids, so one running maximum per chunk tells whether any of its
// 16 steps landed in a final state or left the hot rows; if not, the chunk costs what a plain scan costs.
// When a sample showed final states to be frequent (kAlways) that first pass is skipped and every chunk
// is counted.
//
// Where a lane's counts go (Row): the batch kernel's lane-private row of u32 in global memory (of u64, added to, for
// pire_gpu_count_batch_from), or for one string over the grid (CountStringKernel) its warp's row of u32 in shared memory,
// shared by 32 lanes (atomics), or -- too many regexps for such rows -- the caller's u64 counters in global memory.
struct WarpRow {
    uint32_t* shared;               // the warp's row, or null
    unsigned long long* global;     // used when `shared` is null
};

__device__ __forceinline__ void AddTo(uint32_t* row, uint32_t id, uint32_t add) { row[id] += add; }

// the caller's counters, added to: a zero add reads and writes nothing
__device__ __forceinline__ void AddTo(unsigned long long* row, uint32_t id, uint32_t add)
{
    if (add)
        row[id] += add;
}

__device__ __forceinline__ void AddTo(const WarpRow& row, uint32_t id, uint32_t add)
{
    if (add == 0)
        return;
    if (row.shared)
        atomicAdd(row.shared + id, add);
    else
        atomicAdd(row.global + id, (unsigned long long) add);
}

template <int kWords, class Row = uint32_t*>
struct Counter {
    uint64_t a8[kWords];            // 8 x 8 bits: at most 16 steps x 15 per field between Widen() calls
    uint64_t even[kWords], odd[kWords];   // 4 x 16 bits each
    uint32_t groups;
    Row row;
    const uint64_t* hot_w;          // shared: (H + 1) * kWords words, the sink's are zero
    const uint64_t* all_w;          // global: states * kWords

    __device__ __forceinline__ void Reset(const ScanArgs& a, const uint64_t* hot_weights, Row r)
    {
#pragma unroll
        for (int j = 0; j < kWords; ++j)
            a8[j] = even[j] = odd[j] = 0;
        groups = 0;
        row = r;
        hot_w = hot_weights;
        all_w = a.weights;
    }
    __device__ __forceinline__ void Step(const ScanArgs&, uint32_t H, uint32_t s)          // TakeAction
    {
#pragma unroll
        for (int j = 0; j < kWords; ++j)
            a8[j] += s < H ? hot_w[s * kWords + j] : __ldg(all_w + (size_t) s * kWords + j);
    }
    __device__ __forceinline__ void Flush(uint32_t regexps)
    {
#pragma unroll
        for (int j = 0; j < kWords; ++j) {
            for (uint32_t f = 0; f < 8 && j * 8 + f < regexps; ++f) {
                const uint64_t src = (f & 1) ? odd[j] : even[j];
                const uint32_t add = (uint32_t) (src >> (16 * (f >> 1))) & 0xffffu;
                if (add)
                    AddTo(row, j * 8 + f, add);
            }
            even[j] = odd[j] = 0;
        }
        groups = 0;
    }
    __device__ __forceinline__ void EndGroup(uint32_t regexps)      // after at most 16 steps
    {
#pragma unroll
        for (int j = 0; j < kWords; ++j) {
            even[j] += a8[j] & 0x00FF00FF00FF00FFull;
            odd[j] += (a8[j] >> 8) & 0x00FF00FF00FF00FFull;
            a8[j] = 0;
        }
        if (++groups >= 120)                                        // 120 x 16 x 15 < 65536
            Flush(regexps);
    }
    __device__ __forceinline__ void Discard()
    {
#pragma unroll
        for (int j = 0; j < kWords; ++j)
            a8[j] = 0;
    }
    __device__ __forceinline__ void Finish(uint32_t regexps) { Flush(regexps); }
};

template <class Row>
struct Counter<0, Row> {
    uint32_t c0, c1, c2, c3;
    Row row;

    __device__ __forceinline__ void Reset(const ScanArgs&, const uint64_t*, Row r)
    {
        c0 = c1 = c2 = c3 = 0;
        row = r;
    }
    __device__ __forceinline__ void Step(const ScanArgs& a, uint32_t H, uint32_t s)
    {
        const bool final = s < H ? s >= a.first_final_hot : (__ldg(a.flags + s) & 1u) != 0;
        if (!final)
            return;
        uint32_t k = __ldg(a.acc_begin + s);
        const uint32_t e = __ldg(a.acc_begin + s + 1);
        for (; k < e; ++k) {
            const uint32_t id = __ldg(a.acc_ids + k);
            c0 += id == 0;
            c1 += id == 1;
            c2 += id == 2;
            c3 += id == 3;
            if (id >= 4)
                AddTo(row, id, 1);
        }
    }
    __device__ __forceinline__ void EndGroup(uint32_t) {}
    __device__ __forceinline__ void Discard() {}
    __device__ __forceinline__ void Finish(uint32_t regexps)
    {
        AddTo(row, 0, c0);
        if (regexps > 1) AddTo(row, 1, c1);
        if (regexps > 2) AddTo(row, 2, c2);
        if (regexps > 3) AddTo(row, 3, c3);
    }
};

template <int kWords, bool kAlways, class Row>
__device__ __forceinline__ void CountChunk16(const ScanArgs& a, const Tables& t, LaneState& s, uint4 v, Counter<kWords, Row>& c)
{
    const uint32_t before = s.g;
    if (!kAlways || kWords == 0) {
        uint32_t g = before, top = 0;
#pragma unroll
        for (int w = 0; w < 4; ++w) {
            const uint32_t word = w == 0 ? v.x : w == 1 ? v.y : w == 2 ? v.z : v.w;
            FastStep<false>(t, g, word, 0x5540);
            top = max(top, g);
            FastStep<false>(t, g, word, 0x5541);
            top = max(top, g);
            FastStep<false>(t, g, word, 0x5542);
            top = max(top, g);
            FastStep<false>(t, g, word, 0x5543);
            top = max(top, g);
        }
        if (top < a.first_final_hot) {       // sixteen steps through non-final hot states: nothing to count
            s.g = g;
            return;
        }
    }
    if (kWords > 0 && before != t.H) {
        // the chunk again (or, kAlways, for the first time) with the packed increments of every state entered
        uint32_t g = before;
#pragma unroll
        for (int w = 0; w < 4; ++w) {
            const uint32_t word = w == 0 ? v.x : w == 1 ? v.y : w == 2 ? v.z : v.w;
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                FastStep<false>(t, g, word, 0x5540 + b);
                c.Step(a, 0xffffffffu, g);              // g <= H: always the shared copy
            }
        }
        if (g != t.H) {
            c.EndGroup(a.regexps);
            s.g = g;
            return;
        }
        // left the hot rows somewhere inside: forget what was added (the sink's increments are zero, but
        // the steps after the miss were not the real ones) and replay through the complete table
        c.Discard();
    }
    uint32_t full = before == t.H ? s.cold : before;
    EdgeBytes eb(v, 0);
    for (int k = 0; k < 16; ++k) {
        full = SlowStep(t, full, eb.Next());
        c.Step(a, t.H, full);
    }
    c.EndGroup(a.regexps);
    SetFull(t, s, full);
}

// The entries of the states a walk enters: counted (kWrite false: n is the count), or written from index n on, up to
// index `stop` (kWrite: the end of the lane's slice or the capacity).
template <bool kWrite>
struct EndsSink {
    uint64_t n;
    uint64_t stop;

    __device__ __forceinline__ bool Full() const { return kWrite && n >= stop; }
    // s a full state, entered when `pos` bytes of the call's text had been consumed
    __device__ __forceinline__ void Take(const ScanArgs& a, const Tables& t, uint32_t s, uint64_t pos)
    {
        const bool final = s < t.H ? s >= a.first_final_hot : (__ldg(a.flags + s) & 1u) != 0;
        if (!final)
            return;
        uint32_t k = __ldg(a.acc_begin + s);
        const uint32_t e = __ldg(a.acc_begin + s + 1);
        if (!kWrite) {
            n += e - k;
            return;
        }
        for (; k < e && n < stop; ++k, ++n) {
            if (a.ends)
                a.ends[n] = a.ends_base + pos;
            if (a.ids)
                a.ids[n] = __ldg(a.acc_ids + k);
        }
    }
};

// 16 bytes at position `at` of the text.  Counting adds the hot list lengths of a chunk that stays in the hot rows
// without a table read per step; writing needs each final state's list, so it takes every chunk with a final state
// through the complete table (whose hot rows are the shared ones, SlowStep).
template <bool kWrite>
__device__ __forceinline__ void EndsChunk16(const ScanArgs& a, const Tables& t, const uint32_t* hot_len, LaneState& s, uint4 v,
                                            uint64_t at, EndsSink<kWrite>& o)
{
    const uint32_t before = s.g;
    uint32_t g = before, top = 0;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
        const uint32_t word = w == 0 ? v.x : w == 1 ? v.y : w == 2 ? v.z : v.w;
        FastStep<false>(t, g, word, 0x5540);
        top = max(top, g);
        FastStep<false>(t, g, word, 0x5541);
        top = max(top, g);
        FastStep<false>(t, g, word, 0x5542);
        top = max(top, g);
        FastStep<false>(t, g, word, 0x5543);
        top = max(top, g);
    }
    if (top < a.first_final_hot) {           // sixteen steps through non-final hot states: no entry
        s.g = g;
        return;
    }
    if (!kWrite && top < t.H) {
        // every step in the hot rows (the sink is the highest id), some in final ones: their list lengths
        uint32_t add = 0;
        g = before;
#pragma unroll
        for (int w = 0; w < 4; ++w) {
            const uint32_t word = w == 0 ? v.x : w == 1 ? v.y : w == 2 ? v.z : v.w;
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                FastStep<false>(t, g, word, 0x5540 + b);
                add += hot_len[g];
            }
        }
        o.n += add;
        s.g = g;
        return;
    }
    uint32_t full = before == t.H ? s.cold : before;
    EdgeBytes eb(v, 0);
    for (int k = 0; k < 16; ++k) {
        full = SlowStep(t, full, eb.Next());
        o.Take(a, t, full, at + k + 1);
    }
    SetFull(t, s, full);
}

// CountWalk reports every state it enters to a sink: a Counter (counting), or an EndsSink (where the matches of
// a batch end), which also takes the position of the state: `pos`, or `at` for the first byte of a chunk, is the string's
// base in its stream plus the bytes consumed.  A Counter ignores the position.
template <int kWords, class Row>
__device__ __forceinline__ void SinkTake(const ScanArgs& a, const Tables& t, Counter<kWords, Row>& c, uint32_t s, uint64_t)
{
    c.Step(a, t.H, s);
}
template <bool kWrite>
__device__ __forceinline__ void SinkTake(const ScanArgs& a, const Tables& t, EndsSink<kWrite>& o, uint32_t s, uint64_t pos)
{
    o.Take(a, t, s, pos);
}
template <int kWords, class Row>
__device__ __forceinline__ void SinkGroup(const ScanArgs& a, Counter<kWords, Row>& c) { c.EndGroup(a.regexps); }
template <bool kWrite>
__device__ __forceinline__ void SinkGroup(const ScanArgs&, EndsSink<kWrite>&) {}
template <int kWords, class Row>
__device__ __forceinline__ bool SinkFull(const Counter<kWords, Row>&) { return false; }
template <bool kWrite>
__device__ __forceinline__ bool SinkFull(const EndsSink<kWrite>& o) { return o.Full(); }
template <int kWords, bool kAlways, class Row>
__device__ __forceinline__ void SinkChunk16(const ScanArgs& a, const Tables& t, const uint32_t*, LaneState& s, uint4 v, uint64_t,
                                            Counter<kWords, Row>& c)
{
    CountChunk16<kWords, kAlways>(a, t, s, v, c);
}
template <int kWords, bool kAlways, bool kWrite>
__device__ __forceinline__ void SinkChunk16(const ScanArgs& a, const Tables& t, const uint32_t* hot_len, LaneState& s, uint4 v,
                                            uint64_t at, EndsSink<kWrite>& o)
{
    EndsChunk16<kWrite>(a, t, hot_len, s, v, at, o);
}

// kFrom (pire_gpu_count_batch_from): string i's counts are added to its row of u64 in a.counts64, its walk starts from
// a.starts[i] when a.starts is given (StartFrom; that state is not counted again; read before anything writes string i's
// state, so a.starts may be a.state_idx), and its last state is reported through a.fin.  A start outside the scanner walks
// nothing, counts nothing and reports match 0 and state 0xFFFFFFFF; the lane carries it as kUnknownStart in `full`
// rather than in a flag of its own, which would stay live through the walk.
constexpr uint32_t kUnknownStart = 0xFFFFFFFFu;

// The walk of CountKernel, and with Ends an EndsSink (kFrom, kWords 0) that of MatchEndsBatchKernel
// (pire_gpu_match_ends_batch_from), in two launches on either side of a scan (LaunchMatchEndsBatch).  EndsSink<false> counts string i's entries into a.entry_counts[i + 1] and
// leaves its state before EndMark (or kUnknownStart) in a.last_states[i]; it writes no output, so that the second walk
// still reads the caller's start and base.  EndsSink<true> walks string i again when its slice [a.entry_first[i],
// a.entry_first[i + 1]) begins below the capacity, and writes it up to its end or the capacity; then string i's match
// bit, its state (from a.last_states) and a.pos[i] + its length, and string 0's lane the new *a.found.
// `a` by value, as the kernels take it: so the counting kernels compile to what they did when this was their own body.
template <int kWords, bool kAlways, bool kFrom, class Ends>
__device__ __forceinline__ void CountWalk(const ScanArgs a)
{
    constexpr bool kEnds = !std::is_void_v<Ends>;
    constexpr bool kWrite = std::is_same_v<Ends, EndsSink<true>>;
    uint8_t* const smem = pire_b200_smem;
    SharedView sv = CarveShared(smem, a.hot);
    StageTables(a, sv, a.hot8, a.hot);
    // packed increments of the hot states (and zeros for the sink) behind the staging ring
    uint64_t* const hot_w = reinterpret_cast<uint64_t*>(sv.stage + kStageBytes);
    if (kWords > 0) {
        for (uint32_t i = threadIdx.x; i < (a.hot + 1) * kWords; i += blockDim.x)
            hot_w[i] = i < a.hot * kWords ? a.weights[i] : 0;
        __syncthreads();
    }
    // the counting ends walk: in the same place, the accept-list length of every hot state (0 for the non-final ones)
    uint32_t* const hot_len = reinterpret_cast<uint32_t*>(sv.stage + kStageBytes);
    if (kEnds && !kWrite) {
        for (uint32_t i = threadIdx.x; i < a.hot; i += blockDim.x)
            hot_len[i] = i >= a.first_final_hot ? __ldg(a.acc_begin + i + 1) - __ldg(a.acc_begin + i) : 0u;
        __syncthreads();
    }

    Tables t;
    t.hot = sv.hot;
    t.base = SmemAddr(sv.hot);
    t.cls = sv.cls;
    t.full = a.full;
    t.H = a.hot;
    t.letters = a.letters;
    t.wide = a.wide;
    t.m0 = 0;

    const uint32_t lane = threadIdx.x & 31;
    const uint64_t units = (a.n + 31) / 32;
    const uint64_t warps = (uint64_t) gridDim.x * kWarpsPerBlock;
    const uint32_t stage = SmemAddr(sv.stage) + (((threadIdx.x >> 5) * kStageSlots) * 32 + lane) * 16;
    const uintptr_t buf_lo = reinterpret_cast<uintptr_t>(a.corpus);
    const uintptr_t buf_hi = buf_lo + (a.offsets ? a.offsets[a.n] - a.trim : a.n * a.fixed_len);

    for (uint64_t unit = (uint64_t) blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5); unit < units; unit += warps) {
        const uint64_t i = unit * 32 + lane;
        const bool valid = i < a.n;
        uint64_t b = 0, e = 0;
        if (valid) {
            if (a.offsets) {
                b = a.offsets[i];
                e = a.offsets[i + 1] - a.trim;
                e = e < b ? b : e;       // an empty entry of a trimmed (lines) batch, or caller offsets that step back
            } else {
                b = i * a.fixed_len;
                e = b + a.fixed_len;
            }
        }
        using Row = std::conditional_t<kFrom, unsigned long long*, uint32_t*>;
        std::conditional_t<kEnds, Ends, Counter<kWords, Row>> c;
        uint32_t full = a.initial;
        const uint64_t bytes = e - b;                               // kEnds: the string's length
        uint64_t base = 0;                                          // kEnds: the position of the string's first byte
        if constexpr (kEnds) {
            c.n = c.stop = 0;
            if (valid) {
                base = a.pos ? a.pos[i] : 0;
                if (kWrite) {
                    // the slice, cut at the capacity; a string with nothing to write there walks no byte
                    const uint64_t to = a.entry_first[i + 1];
                    c.n = a.entry_first[i];
                    c.stop = to < a.ends_capacity ? to : a.ends_capacity;
                    if (c.n >= c.stop)
                        e = b;
                }
            }
        } else if constexpr (kFrom) {
            c.Reset(a, hot_w, a.counts64 + (valid ? i : 0) * a.regexps);
        } else {
            c.Reset(a, hot_w, a.counts + (valid ? i : 0) * a.regexps);
        }
        if constexpr (kFrom) {
            if (valid && a.starts) {
                bool known;
                StartFrom(a, t, a.starts[i], full, known);          // BeginMark stepped when a.with_begin
                if (!known) {
                    full = kUnknownStart;                           // no byte is walked, so it is still there at the end
                    e = b;
                }
            }
        }
        if constexpr (kWrite) {
            if (valid && a.strings)                                 // after the reads of the start and the base
                for (uint64_t k = c.n; k < c.stop; ++k)
                    a.strings[k] = (uint32_t) i;
        }
        const uint8_t* p = a.corpus + b;
        const uint8_t* end = a.corpus + e;
        const uint8_t* const str = p;

        if (valid) {
            if (kFrom && a.starts) {
                if (full != kUnknownStart && a.with_begin)
                    SinkTake(a, t, c, full, base);                  // the state Step(BeginMark) reached
            } else {
                SinkTake(a, t, c, full, base);                      // Initialize ends in TakeAction, half_final.h:136-141
                if (a.with_begin) {
                    full = FullNext(t, full, a.begin_class);        // Step(BeginMark), run.h:50-57
                    SinkTake(a, t, c, full, base);
                }
            }
            SinkGroup(a, c);
        }
        {
            const uint32_t misalign = (uint32_t) (reinterpret_cast<uintptr_t>(p) & 15);
            if (p < end && misalign != 0) {
                const uint64_t room = (uint64_t) (end - p);
                const uint32_t nhead = room < 16 - misalign ? (uint32_t) room : 16 - misalign;
                const uint8_t* chunk = p - misalign;
                if (reinterpret_cast<uintptr_t>(chunk) >= buf_lo && reinterpret_cast<uintptr_t>(chunk) + 16 <= buf_hi) {
                    EdgeBytes eb(LoadEdge16(chunk), misalign);
                    for (uint32_t k = 0; k < nhead; ++k) {
                        full = SlowStep(t, full, eb.Next());
                        SinkTake(a, t, c, full, base + k + 1);
                    }
                } else {
                    for (uint32_t k = 0; k < nhead; ++k) {
                        full = SlowStep(t, full, p[k]);
                        SinkTake(a, t, c, full, base + k + 1);
                    }
                }
                SinkGroup(a, c);
                p += nhead;
            }
        }
        LaneState s;
        SetFull(t, s, full);
        if (a.uniform) {
            // fixed-length, 32-byte aligned batch: 32-byte loads ping-pong through registers, no staging ring (see PrefixKernel)
            const uint32_t len = (uint32_t) (end - p);
            if (len != 0) {
                const uint64_t at = base + (uint64_t) (p - str);
                uint4 a0, a1, b0, b1;
                LoadStream32(p, a0, a1);
                for (uint32_t off = 0;;) {
                    off += 32;
                    const bool more_b = off < len;
                    if (more_b)
                        LoadStream32(p + off, b0, b1);
                    SinkChunk16<kWords, kAlways>(a, t, hot_len, s, a0, at + off - 32, c);
                    SinkChunk16<kWords, kAlways>(a, t, hot_len, s, a1, at + off - 16, c);
                    if (!more_b || SinkFull(c))
                        break;
                    off += 32;
                    const bool more_a = off < len;
                    if (more_a)
                        LoadStream32(p + off, a0, a1);
                    SinkChunk16<kWords, kAlways>(a, t, hot_len, s, b0, at + off - 32, c);
                    SinkChunk16<kWords, kAlways>(a, t, hot_len, s, b1, at + off - 16, c);
                    if (!more_a || SinkFull(c))
                        break;
                }
            }
            p = end;
        }
        const uint32_t chunks = (uint32_t) ((end - p) >> 4);
        const uint64_t at = base + (uint64_t) (p - str);
#pragma unroll
        for (int j = 0; j < kStageSlots; ++j) {
            if ((uint32_t) j < chunks)
                CopyAsync16(stage + j * 512, p + 16 * j);
            CopyAsyncCommit();
        }
        for (uint32_t k = 0; __any_sync(0xffffffffu, k < chunks); k += kStageSlots) {
#pragma unroll
            for (int j = 0; j < kStageSlots; ++j) {
                CopyAsyncWait<kStageSlots - 1>();
                const uint4 v = LoadShared16(stage + j * 512);
                if (k + kStageSlots + j < chunks)
                    CopyAsync16(stage + j * 512, p + 16 * (size_t) (k + kStageSlots + j));
                CopyAsyncCommit();
                if (k + j < chunks && !SinkFull(c))
                    SinkChunk16<kWords, kAlways>(a, t, hot_len, s, v, at + 16 * (uint64_t) (k + j), c);
            }
        }
        CopyAsyncWait<0>();
        full = FullState(t, s);
        p += 16 * (size_t) chunks;
        if (p < end) {
            const uint32_t ntail = (uint32_t) (end - p);
            const uint64_t at = base + (uint64_t) (p - str);
            if (reinterpret_cast<uintptr_t>(p) + 16 <= buf_hi) {
                EdgeBytes eb(LoadEdge16(p), 0);
                for (uint32_t k = 0; k < ntail; ++k) {
                    full = SlowStep(t, full, eb.Next());
                    SinkTake(a, t, c, full, at + k + 1);
                }
            } else {
                for (uint32_t k = 0; k < ntail; ++k) {
                    full = SlowStep(t, full, p[k]);
                    SinkTake(a, t, c, full, at + k + 1);
                }
            }
        }
        if constexpr (kEnds) {
            if (valid && full != kUnknownStart && a.through_end)
                SinkTake(a, t, c, FullNext(t, full, a.end_class), base + bytes);   // Step(EndMark)
            if constexpr (!kWrite) {
                if (valid) {
                    a.entry_counts[i + 1] = c.n;
                    a.last_states[i] = full;
                    if (i == 0)
                        a.entry_counts[0] = *a.found;           // the only read of *a.found: the scan starts from it
                }
            } else {
                const uint32_t last = valid ? a.last_states[i] : kUnknownStart;
                const bool known = last != kUnknownStart;
                const DeviceFin f = known ? a.fin[last] : DeviceFin{0u, 0u};
                const unsigned matched = __ballot_sync(0xffffffffu, (f.result >> 31) != 0);
                if (a.match_bits && lane == 0)
                    a.match_bits[unit] = matched;
                if (valid) {
                    if (a.state_idx)
                        a.state_idx[i] = known ? f.result & 0x7fffffffu : 0xFFFFFFFFu;
                    if (a.pos)
                        a.pos[i] = base + bytes;
                    if (i == 0)
                        *a.found = a.entry_first[a.n];
                }
            }
        } else if constexpr (kFrom) {
            // a.fin is the table of the call's marks: the state before EndMark is its index
            const bool known = full != kUnknownStart;
            if (valid && known && a.through_end)
                c.Step(a, t.H, FullNext(t, full, a.end_class));     // Step(EndMark)
            c.EndGroup(a.regexps);
            const DeviceFin f = valid && known ? a.fin[full] : DeviceFin{0u, 0u};
            const unsigned matched = __ballot_sync(0xffffffffu, (f.result >> 31) != 0);
            if (a.match_bits && lane == 0)
                a.match_bits[unit] = matched;
            if (valid) {
                if (a.state_idx)
                    a.state_idx[i] = known ? f.result & 0x7fffffffu : 0xFFFFFFFFu;
                c.Finish(a.regexps);
            }
        } else {
            if (valid && a.through_end) {
                full = FullNext(t, full, a.end_class);               // Step(EndMark)
                c.Step(a, t.H, full);
            }
            c.EndGroup(a.regexps);
            const bool final = valid && (__ldg(a.flags + full) & 1u) != 0;
            const unsigned matched = __ballot_sync(0xffffffffu, final);
            if (a.match_bits && lane == 0)
                a.match_bits[unit] = matched;
            if (valid)
                c.Finish(a.regexps);
        }
    }
}

template <int kWords, bool kAlways, bool kFrom = false>
__global__ void __launch_bounds__(kBlock, kGenericBlocksPerSM) CountKernel(const __grid_constant__ ScanArgs a)
{
    CountWalk<kWords, kAlways, kFrom, void>(a);
}

// pire_gpu_match_ends_batch_from: the counting walk (kWrite false) and the writing walk of LaunchMatchEndsBatch
template <bool kWrite>
__global__ void __launch_bounds__(kBlock, kGenericBlocksPerSM) MatchEndsBatchKernel(const __grid_constant__ ScanArgs a)
{
    CountWalk<0, false, true, EndsSink<kWrite>>(a);
}

// ---------------------------------------------------------------- counting one string over the whole grid
//
// HalfFinalScanner counts of one string (pire_gpu_count_string).  The counts depend on every state the walk enters, so
// each lane needs the true state at the start of its piece; the kernel runs in two phases in one cooperative launch.
//   1. Locate: ScanStringKernel's head, pieces, walk and stitch (WalkPiece, PIRE_B200_STITCH_GRID), with the plain walk.  After its last
//      grid.sync() every lane knows the true state at the start of its piece.
//   2. Count: every lane walks its piece again from there with CountChunk16, 32-byte loads one block ahead in registers
//      (CountKernel's uniform body).  The head (before the first 32-byte boundary), Initialize() and BeginMark are counted
//      by the grid's first lane, the tail and EndMark by its last lane: once each, through the complete table.
// Counters: every lane keeps CountKernel's registers and flushes them into its warp's row of u32 in shared memory (shared
// atomics, one flush per 120 chunks).  A warp walks at most 80 GB / 4 224 warps (19 MB) of an H100's memory, 15 per byte
// at most, well inside 32 bits.  At the end every CTA adds its warps' rows into the caller's u64 counters with one 64-bit
// atomic per regexp.  With more regexps than kCountRowsMax the rows do not fit; flushes then go to the u64 counters.
// The plain walk locates: it is the one AUTO runs for pire_gpu_run_string on every automaton (ResolveVariant, non-uniform),
// and the counting walk is plain as well, so the two phases share their code shape.
template <int kWords, bool kAlways>
__global__ void __launch_bounds__(kBlock, kStringBlocksPerSM) CountStringKernel(const __grid_constant__ ScanArgs a)
{
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    uint8_t* const smem = pire_b200_smem;
    SharedView sv = CarveShared(smem, a.hot);
    StageTables(a, sv, a.hot8, a.hot);
    // behind the marks: the hot states' packed increments (zeros for the sink), then every warp's row of counters
    uint64_t* const hot_w = reinterpret_cast<uint64_t*>(sv.stage + kSplitMarkBytes);
    uint32_t* const rows = reinterpret_cast<uint32_t*>(hot_w + (size_t) (a.hot + 1) * kWords);
    if (kWords > 0)
        for (uint32_t i = threadIdx.x; i < (a.hot + 1) * kWords; i += blockDim.x)
            hot_w[i] = i < a.hot * kWords ? a.weights[i] : 0;
    if (a.count_rows)
        for (uint32_t i = threadIdx.x; i < kWarpsPerBlock * a.regexps; i += blockDim.x)
            rows[i] = 0;
    __syncthreads();

    Tables t;
    t.hot = sv.hot;
    t.base = SmemAddr(sv.hot);
    t.cls = sv.cls;
    t.full = a.full;
    t.H = a.hot;
    t.letters = a.letters;
    t.wide = a.wide;
    t.m0 = a.exit_bitmap0;

    // the true start, as in ScanStringKernel (*a.start_idx may be the output word: written only after the last grid.sync())
    uint32_t start = a.start;
    bool valid = true;
    if (a.start_idx)
        StartFrom(a, t, *a.start_idx, start, valid);
    const bool skip = !valid || (start < t.H && sv.noexit[start] != 0);       // multi.h:955-958: no byte leaves it

    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warp = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const uint32_t warps = gridDim.x * kWarpsPerBlock;
    uint8_t* const marks = sv.stage + (threadIdx.x >> 5) * (32 * kSplitMarks) + lane;
    const uintptr_t buf_lo = reinterpret_cast<uintptr_t>(a.corpus);
    const uintptr_t buf_hi = buf_lo + a.fixed_len;
    const uint8_t* const end = a.corpus + a.fixed_len;

    // phase 1, locate: the head by the grid's first warp, then the pieces (ScanStringKernel)
    LaneState s;
    SetFull(t, s, start);
    if (warp == 0 && !skip) {
        const uint8_t* p = a.corpus;
        const uint32_t mis = (uint32_t) (buf_lo & 15);
        if (p < end && mis != 0) {
            const uint64_t room = (uint64_t) (end - p);
            const uint32_t nhead = room < 16 - mis ? (uint32_t) room : 16 - mis;
            EdgeFast<false>(t, s, EdgeBytes(LoadChunk16(p - mis, buf_lo, buf_hi), mis).Words(), nhead);
            p += nhead;
        }
        if ((reinterpret_cast<uintptr_t>(p) & 16) && end - p >= 16)
            Chunk16<false>(t, s, LoadEdge16(p));
    }
    const uint8_t* const body = StringBody(a.corpus, end);
    const uint32_t blocks_total = (reinterpret_cast<uintptr_t>(body) & 31) ? 0u : (uint32_t) ((end - body) >> 5);
    const uint32_t lanes = gridDim.x * kBlock;
    const uint32_t me = blockIdx.x * kBlock + threadIdx.x;
    const uint32_t base = blocks_total / lanes, rem = blocks_total % lanes;
    const uint32_t my_blocks = base + (me < rem ? 1u : 0u);
    const uint64_t my_first = (uint64_t) me * base + (me < rem ? me : rem);
    const uint32_t trips = base + (rem ? 1u : 0u);
    const uint32_t per_mark = (trips + kSplitMarks - 1) / kSplitMarks;
    const uint8_t* const piece = body + 32 * my_first;
    const uint32_t first_start = __shfl_sync(0xffffffffu, FullState(t, s), 0);

    uint32_t start_full = me == 0 ? first_start : 0u;
    uint32_t end_full = start_full;
    if (!skip) {
        SetFull(t, s, start_full);
        WalkPiece<false>(t, s, piece, my_blocks, trips, per_mark, marks, 0);
        end_full = FullState(t, s);

        uint4 head0 = make_uint4(0, 0, 0, 0), head1 = head0;
        bool head_fresh = my_blocks != 0;
        if (head_fresh)
            LoadStream32P(piece, head0, head1);
        PIRE_B200_STITCH_GRID(false);
    } else {
        grid.sync();
    }
    if (!valid) {
        // a start outside the scanner reads no table and counts nothing: match 0, state 0xFFFFFFFF
        if (me == lanes - 1) {
            if (a.match_bits)
                a.match_bits[0] = 0;
            if (a.state_idx)
                a.state_idx[0] = 0xFFFFFFFFu;
        }
        return;
    }
    if (skip)
        start_full = start;  // a NoExit start: every piece starts (and stays) there, and each of its steps is counted

    // phase 2, count
    Counter<kWords, WarpRow> c;
    c.Reset(a, hot_w, WarpRow{a.count_rows ? rows + (threadIdx.x >> 5) * a.regexps : nullptr, a.counts64});
    if (me == 0) {
        // Initialize() ends in TakeAction (half_final.h:136-141); a resumed run counted its start in the previous call.
        // `start` is the state after BeginMark when it was asked for.
        if (!a.start_idx)
            c.Step(a, t.H, a.initial);
        if (a.with_begin)
            c.Step(a, t.H, start);
        c.EndGroup(a.regexps);
        uint32_t full = start;
        for (const uint8_t* p = a.corpus; p < body; ++p) {
            full = SlowStep(t, full, *p);
            c.Step(a, t.H, full);
            c.EndGroup(a.regexps);
        }
    }
    SetFull(t, s, start_full);
    if (my_blocks != 0) {
        const uint32_t len = 32u * my_blocks;
        uint4 a0, a1, b0, b1;
        LoadStream32(piece, a0, a1);
        for (uint32_t off = 0;;) {
            off += 32;
            const bool more_b = off < len;
            if (more_b)
                LoadStream32(piece + off, b0, b1);
            CountChunk16<kWords, kAlways>(a, t, s, a0, c);
            CountChunk16<kWords, kAlways>(a, t, s, a1, c);
            if (!more_b)
                break;
            off += 32;
            const bool more_a = off < len;
            if (more_a)
                LoadStream32(piece + off, a0, a1);
            CountChunk16<kWords, kAlways>(a, t, s, b0, c);
            CountChunk16<kWords, kAlways>(a, t, s, b1, c);
            if (!more_a)
                break;
        }
    }
    if (me == lanes - 1) {
        // the tail from the last piece's end, EndMark, and the results (those of ScanStringKernel)
        uint32_t last = FullState(t, s);
        for (const uint8_t* p = body + 32 * (size_t) blocks_total; p < end; ++p) {
            last = SlowStep(t, last, *p);
            c.Step(a, t.H, last);
            c.EndGroup(a.regexps);
        }
        if (a.through_end) {
            c.Step(a, t.H, FullNext(t, last, a.end_class));          // Step(EndMark)
            c.EndGroup(a.regexps);
        }
        const DeviceFin f = a.fin[last];
        if (a.match_bits)
            a.match_bits[0] = f.result >> 31;
        if (a.state_idx)
            a.state_idx[0] = f.result & 0x7fffffffu;
    }
    c.Finish(a.regexps);
    if (!a.count_rows)
        return;
    __syncthreads();
    for (uint32_t id = threadIdx.x; id < a.regexps; id += blockDim.x) {
        unsigned long long sum = 0;
        for (uint32_t w = 0; w < kWarpsPerBlock; ++w)
            sum += rows[w * a.regexps + id];
        if (sum)
            atomicAdd(a.counts64 + id, sum);
    }
}

// ---------------------------------------------------------------- where the matches end in one string over the whole grid
//
// pire_gpu_match_ends_string: every TakeAction of HalfFinalScanner (half_final.h:154-163) on one string as entries
// (position, regexp id), in walk order.  One cooperative launch of CountStringKernel's grid and pieces, in four phases:
//   1. Locate: CountStringKernel's phase 1 unchanged.  After its last grid.sync() every lane knows the true state at the
//      start of its piece.
//   2. Count: every lane walks its piece from there and counts its entries (EndsLane<false>).  A 16-step running maximum
//      of hot ids skips every chunk that enters no final state (CountChunk16's test); a chunk that does is walked again
//      through the hot rows, adding the list lengths staged in shared memory, or through the complete table when it
//      leaves the hot rows.  The grid's first lane adds Initialize(), BeginMark and the head, its last lane the tail and
//      EndMark, and the last lane reports the match and the state.
//   3. Scan: an exclusive prefix sum of the lane totals in lane order, which is the order of the text, over the grid: a
//      block scan, every CTA's total published to scratch, grid.sync(), every CTA adds up the totals of the CTAs before it.
//   4. Emit: every lane whose slice begins below the capacity walks its piece once more (EndsLane<true>) and writes its
//      entries into its slice, up to its last entry or the capacity, whichever comes first.
// The scan places the entries, where atomics appending them would not: the arrays are the same on every run, and a
// buffer too small for the answer holds its first `capacity` entries.

// One lane's share of the string, walked by phase 2 (kWrite false) and again by phase 4 (kWrite): Initialize(),
// BeginMark and the head (the grid's first lane), the piece from its true start `start_full`, the tail and EndMark (the
// last lane).  Returns the state after the lane's bytes (before EndMark).  A writing walk stops when its sink is full.
template <bool kWrite>
__device__ __forceinline__ uint32_t EndsLane(const ScanArgs& a, const Tables& t, const uint32_t* hot_len, uint32_t start,
                                             uint32_t start_full, bool first, bool last, const uint8_t* body,
                                             const uint8_t* piece, uint32_t my_blocks, EndsSink<kWrite>& o)
{
    const uint8_t* const end = a.corpus + a.fixed_len;
    if (first) {
        // Initialize() ends in TakeAction (half_final.h:136-141); a resumed run reported its start in the previous call.
        // `start` is the state after BeginMark when it was asked for.
        if (!a.start_idx)
            o.Take(a, t, a.initial, 0);
        if (a.with_begin)
            o.Take(a, t, start, 0);
        uint32_t full = start;
        for (const uint8_t* p = a.corpus; p < body; ++p) {
            full = SlowStep(t, full, *p);
            o.Take(a, t, full, (uint64_t) (p - a.corpus) + 1);
        }
    }
    LaneState s;
    SetFull(t, s, start_full);
    if (my_blocks != 0 && !o.Full()) {
        // CountStringKernel's loop: 32-byte loads one block ahead in registers
        const uint32_t len = 32u * my_blocks;
        const uint64_t at = (uint64_t) (piece - a.corpus);
        uint4 a0, a1, b0, b1;
        LoadStream32(piece, a0, a1);
        for (uint32_t off = 0;;) {
            off += 32;
            const bool more_b = off < len;
            if (more_b)
                LoadStream32(piece + off, b0, b1);
            EndsChunk16<kWrite>(a, t, hot_len, s, a0, at + off - 32, o);
            EndsChunk16<kWrite>(a, t, hot_len, s, a1, at + off - 16, o);
            if (!more_b || o.Full())
                break;
            off += 32;
            const bool more_a = off < len;
            if (more_a)
                LoadStream32(piece + off, a0, a1);
            EndsChunk16<kWrite>(a, t, hot_len, s, b0, at + off - 32, o);
            EndsChunk16<kWrite>(a, t, hot_len, s, b1, at + off - 16, o);
            if (!more_a || o.Full())
                break;
        }
    }
    uint32_t full = FullState(t, s);
    if (last && !o.Full()) {
        for (const uint8_t* p = piece + 32 * (size_t) my_blocks; p < end; ++p) {      // the last piece ends the body
            full = SlowStep(t, full, *p);
            o.Take(a, t, full, (uint64_t) (p - a.corpus) + 1);
        }
        if (a.through_end)
            o.Take(a, t, FullNext(t, full, a.end_class), a.fixed_len);      // Step(EndMark)
    }
    return full;
}

__global__ void __launch_bounds__(kBlock, kStringBlocksPerSM) MatchEndsStringKernel(const __grid_constant__ ScanArgs a)
{
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    uint8_t* const smem = pire_b200_smem;
    SharedView sv = CarveShared(smem, a.hot);
    StageTables(a, sv, a.hot8, a.hot);
    // behind the marks: the scan's words (every warp's entries, the CTA's first entry, *a.found as the call found it),
    // then the accept-list length of every hot state (0 for the non-final ones)
    unsigned long long* const sums = reinterpret_cast<unsigned long long*>(sv.stage + kSplitMarkBytes);
    uint32_t* const hot_len = reinterpret_cast<uint32_t*>(sums + kWarpsPerBlock + 2);
    for (uint32_t i = threadIdx.x; i < a.hot; i += blockDim.x)
        hot_len[i] = i >= a.first_final_hot ? __ldg(a.acc_begin + i + 1) - __ldg(a.acc_begin + i) : 0u;
    if (threadIdx.x == 0)
        sums[kWarpsPerBlock + 1] = *a.found;       // read before the first grid.sync(), written after the last
    __syncthreads();

    Tables t;
    t.hot = sv.hot;
    t.base = SmemAddr(sv.hot);
    t.cls = sv.cls;
    t.full = a.full;
    t.H = a.hot;
    t.letters = a.letters;
    t.wide = a.wide;
    t.m0 = a.exit_bitmap0;

    // the true start, as in ScanStringKernel (*a.start_idx may be the output word: written only after a grid.sync())
    uint32_t start = a.start;
    bool valid = true;
    if (a.start_idx)
        StartFrom(a, t, *a.start_idx, start, valid);
    const bool skip = !valid || (start < t.H && sv.noexit[start] != 0);       // multi.h:955-958: no byte leaves it

    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warp = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    const uint32_t warps = gridDim.x * kWarpsPerBlock;
    uint8_t* const marks = sv.stage + (threadIdx.x >> 5) * (32 * kSplitMarks) + lane;
    const uintptr_t buf_lo = reinterpret_cast<uintptr_t>(a.corpus);
    const uintptr_t buf_hi = buf_lo + a.fixed_len;
    const uint8_t* const end = a.corpus + a.fixed_len;

    // phase 1, locate: CountStringKernel's
    LaneState s;
    SetFull(t, s, start);
    if (warp == 0 && !skip) {
        const uint8_t* p = a.corpus;
        const uint32_t mis = (uint32_t) (buf_lo & 15);
        if (p < end && mis != 0) {
            const uint64_t room = (uint64_t) (end - p);
            const uint32_t nhead = room < 16 - mis ? (uint32_t) room : 16 - mis;
            EdgeFast<false>(t, s, EdgeBytes(LoadChunk16(p - mis, buf_lo, buf_hi), mis).Words(), nhead);
            p += nhead;
        }
        if ((reinterpret_cast<uintptr_t>(p) & 16) && end - p >= 16)
            Chunk16<false>(t, s, LoadEdge16(p));
    }
    const uint8_t* const body = StringBody(a.corpus, end);
    const uint32_t blocks_total = (reinterpret_cast<uintptr_t>(body) & 31) ? 0u : (uint32_t) ((end - body) >> 5);
    const uint32_t lanes = gridDim.x * kBlock;
    const uint32_t me = blockIdx.x * kBlock + threadIdx.x;
    const uint32_t base = blocks_total / lanes, rem = blocks_total % lanes;
    const uint32_t my_blocks = base + (me < rem ? 1u : 0u);
    const uint64_t my_first = (uint64_t) me * base + (me < rem ? me : rem);
    const uint32_t trips = base + (rem ? 1u : 0u);
    const uint32_t per_mark = (trips + kSplitMarks - 1) / kSplitMarks;
    const uint8_t* const piece = body + 32 * my_first;
    const uint32_t first_start = __shfl_sync(0xffffffffu, FullState(t, s), 0);

    uint32_t start_full = me == 0 ? first_start : 0u;
    uint32_t end_full = start_full;
    if (!skip) {
        SetFull(t, s, start_full);
        WalkPiece<false>(t, s, piece, my_blocks, trips, per_mark, marks, 0);
        end_full = FullState(t, s);

        uint4 head0 = make_uint4(0, 0, 0, 0), head1 = head0;
        bool head_fresh = my_blocks != 0;
        if (head_fresh)
            LoadStream32P(piece, head0, head1);
        PIRE_B200_STITCH_GRID(false);
    } else {
        grid.sync();
    }
    if (!valid) {
        // a start outside the scanner reads no table and reports nothing: match 0, state 0xFFFFFFFF, *a.found unchanged
        if (me == lanes - 1) {
            if (a.match_bits)
                a.match_bits[0] = 0;
            if (a.state_idx)
                a.state_idx[0] = 0xFFFFFFFFu;
        }
        return;
    }
    if (skip)
        start_full = start;  // a NoExit start: every piece starts (and stays) there, and each of its steps is reported

    // phase 2, count
    const bool first = me == 0, last = me == lanes - 1;
    EndsSink<false> count{0, 0};
    const uint32_t fin = EndsLane<false>(a, t, hot_len, start, start_full, first, last, body, piece, my_blocks, count);
    if (last) {
        const DeviceFin f = a.fin[fin];
        if (a.match_bits)
            a.match_bits[0] = f.result >> 31;
        if (a.state_idx)
            a.state_idx[0] = f.result & 0x7fffffffu;
    }

    // phase 3, scan: inclusive in the warp, the warps' totals in the CTA, the CTAs' totals over the grid
    uint64_t x = count.n;
#pragma unroll
    for (uint32_t d = 1; d < 32; d <<= 1) {
        const uint64_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d)
            x += y;
    }
    if (lane == 31)
        sums[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
        const uint64_t own = lane < kWarpsPerBlock ? sums[lane] : 0;
        uint64_t w = own;
#pragma unroll
        for (uint32_t d = 1; d < 32; d <<= 1) {
            const uint64_t y = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= d)
                w += y;
        }
        if (lane < kWarpsPerBlock)
            sums[lane] = w - own;                   // the warp's first entry in the CTA
        if (lane == 31)
            __stcg(a.string_sums + blockIdx.x, (unsigned long long) w);
    }
    grid.sync();
    if (threadIdx.x < 32) {
        uint64_t before = 0;
        for (uint32_t c = lane; c < blockIdx.x; c += 32)
            before += __ldcg(a.string_sums + c);
#pragma unroll
        for (uint32_t d = 16; d >= 1; d >>= 1)
            before += __shfl_xor_sync(0xffffffffu, before, d);
        if (lane == 0) {
            const uint64_t found = sums[kWarpsPerBlock + 1];
            sums[kWarpsPerBlock] = found + before;  // the CTA's first entry
            if (blockIdx.x == gridDim.x - 1)
                *a.found = found + before + __ldcg(a.string_sums + blockIdx.x);
        }
    }
    __syncthreads();

    // phase 4, emit: the lane's slice is [first entry, first entry + count.n)
    const uint64_t from = sums[kWarpsPerBlock] + sums[threadIdx.x >> 5] + (x - count.n);
    if (count.n == 0 || from >= a.ends_capacity)
        return;
    EndsSink<true> out{from, from + count.n < a.ends_capacity ? from + count.n : a.ends_capacity};
    EndsLane<true>(a, t, hot_len, start, start_full, first, last, body, piece, my_blocks, out);
}

// Visit counter for pire_gpu_scanner_tune: how many input bytes are consumed in
// each state (new numbering).  Run-length compressed so that a lane resting in
// one state issues one atomic per stay, not one per byte.
__global__ void __launch_bounds__(256) VisitCountKernel(const __grid_constant__ ScanArgs a)
{
    const uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n)
        return;
    uint64_t b, e;
    if (a.offsets) {
        b = a.offsets[i];
        e = a.offsets[i + 1] - a.trim;
        e = e < b ? b : e;
    } else {
        b = i * a.fixed_len;
        e = b + a.fixed_len;
    }
    uint32_t s = a.start;
    unsigned long long run = 0;
    for (uint64_t q = b; q < e; ++q) {
        uint32_t c = a.cls[a.corpus[q]];
        size_t at = (size_t) s * a.letters + c;
        uint32_t ns = a.wide ? static_cast<const uint32_t*>(a.full)[at] : (uint32_t) static_cast<const uint16_t*>(a.full)[at];
        ++run;
        if (ns != s) {
            atomicAdd(&a.visits[s], run);
            run = 0;
            s = ns;
        }
    }
    if (run)
        atomicAdd(&a.visits[s], run);
}

__global__ void __launch_bounds__(256) SynthKernel(const __grid_constant__ SynthParams p, const char* __restrict__ plants, uint8_t* __restrict__ out)
{
    const uint32_t pieces = p.string_len / 16;
    const uint64_t total = p.n_strings * pieces;
    const uint32_t words = p.string_len / 8;
    for (uint64_t idx = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (uint64_t) gridDim.x * blockDim.x) {
        const uint64_t local = idx / pieces;
        const uint32_t piece = (uint32_t) (idx % pieces);
        const uint64_t gi = p.first_string + local;
        uint64_t w0 = SynthWord(p.seed, gi, piece * 2, words);
        uint64_t w1 = SynthWord(p.seed, gi, piece * 2 + 1, words);
        uint32_t off = 0;
        int id = SynthPlant(p, gi, &off);
        if (id >= 0) {
            const uint32_t len = p.plant_off[id + 1] - p.plant_off[id];
            const uint32_t lo = piece * 16, hi = lo + 16;
            const bool touches = (off < hi && off + len > lo) || (p.tail && p.plant_mode[id] == 0 && hi == p.string_len);
            if (touches) {
                uint8_t bytes[16];
                for (int k = 0; k < 8; ++k) {
                    bytes[k] = (uint8_t) (w0 >> (8 * k));
                    bytes[8 + k] = (uint8_t) (w1 >> (8 * k));
                }
                for (uint32_t k = 0; k < 16; ++k)
                    bytes[k] = SynthByte(p, plants, gi, lo + k);
                w0 = w1 = 0;
                for (int k = 0; k < 8; ++k) {
                    w0 |= (uint64_t) bytes[k] << (8 * k);
                    w1 |= (uint64_t) bytes[8 + k] << (8 * k);
                }
            }
        }
        uint4 v = make_uint4((uint32_t) w0, (uint32_t) (w0 >> 32), (uint32_t) w1, (uint32_t) (w1 >> 32));
        *reinterpret_cast<uint4*>(out + local * (uint64_t) p.string_len + (uint64_t) piece * 16) = v;
    }
}

__global__ void __launch_bounds__(256) SynthMixedLengthsKernel(uint64_t seed, uint64_t first, uint64_t n, uint64_t* __restrict__ lengths)
{
    const uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        lengths[i] = SynthMixedLength(seed, first + i);
}

// One warp per string: lanes write consecutive 4-byte cells (coalesced).
__global__ void __launch_bounds__(256) SynthMixedFillKernel(uint64_t seed, uint32_t plant_every, uint64_t first, uint64_t n,
                                                            const uint64_t* __restrict__ offsets, uint8_t* __restrict__ out)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t) gridDim.x * (blockDim.x / 32);
    for (uint64_t i = (uint64_t) blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); i < n; i += warps) {
        const uint64_t b = offsets[i];
        const uint32_t len = (uint32_t) (offsets[i + 1] - b);
        uint32_t* dst = reinterpret_cast<uint32_t*>(out + b);      // offsets are multiples of 4
        for (uint32_t cell = lane; cell < len / 4; cell += 32)
            dst[cell] = SynthMixedCellPlanted(seed, plant_every, first + i, len, cell);
    }
}

// The walk a variant takes in the generic (CSR) kernel, its kMode: 0 plain (PLAIN, PRIV), 1 exit filter (PRED), 2 exit
// filter with one byte of look-ahead (the LOOK variants).  The lines kernels walk with the exit filter for 1 and 2.
int WalkMode(int variant)
{
    if (variant == kVariantPred)
        return 1;
    if (variant == kVariantLook || variant == kVariantLook64 || variant == kVariantLook1 || variant == kVariantLookRing1)
        return 2;
    return 0;
}

// The kernel a batch of one variant runs and its launch shape.
struct BatchKernel {
    const void* fn;
    int block;                  // threads per CTA
    size_t ring_warp_bytes;     // each warp's input ring in shared memory, behind the tables
    uint32_t units_per_step;    // units of 32 strings a warp takes at a time
};

template <typename K>
const void* Fn(K* kernel) { return reinterpret_cast<const void*>(kernel); }

// kStarts: the kernels that start every string from its own state (pire_gpu_run_batch_from).  PRIV has no such kernel:
// with starts it is run as PLAIN.
template <bool kStarts>
BatchKernel BatchKernelOf(int variant, bool uniform)
{
    const int mode = WalkMode(variant);
    if (!uniform)
        return {mode == 2 ? Fn(&ScanGenericKernel<2, kStarts>) : mode == 1 ? Fn(&ScanGenericKernel<1, kStarts>) : Fn(&ScanGenericKernel<0, kStarts>),
                kBlock, 0, 1};
    if (variant == kVariantPriv && !kStarts)
        return {Fn(&ScanUniformPrivKernel), kPrivBlock, 0, 1};
    if (variant == kVariantLook)
        return {kStarts ? Fn(&ScanUniformLookRingFromKernel) : Fn(&ScanUniformLookRingKernel), kRingBlock, kRingWarpBytes, 2};
    if (variant == kVariantLook1)
        return {Fn(&ScanUniformLookKernel<false, 48, true, kStarts>), kLookBlock48, 0, 1};
    if (variant == kVariantLook64)
        return {Fn(&ScanUniformLookKernel<true, 48, false, kStarts>), kLookBlock48, 0, 1};
    if (variant == kVariantLookRing1)
        return {Fn(&ScanUniformLookRing1Kernel<kRing1Slots, kStarts>), kRing1Block, (size_t) kRing1Slots * kRing1SlotBytes, 1};
    return {mode == 1 ? Fn(&ScanUniformKernel<true, kStarts>) : Fn(&ScanUniformKernel<false, kStarts>), kBlock, 0, 1};
}

BatchKernel BatchKernelFor(int variant, bool uniform, bool starts)
{
    return starts ? BatchKernelOf<true>(variant, uniform) : BatchKernelOf<false>(variant, uniform);
}

} // namespace

size_t ScanSharedBytes(uint32_t hot, uint32_t priv_rows) { return PrivBytes(priv_rows) + HotBytes(hot) + 512 + 256 + 16; }
size_t GenericSharedBytes(uint32_t hot) { return ScanSharedBytes(hot, 0) + kStageBytes; }

cudaError_t PrepareScanKernels(int device)
{
    cudaError_t err = cudaSetDevice(device);
    if (err != cudaSuccess)
        return err;
    int optin = 0;
    err = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    if (err != cudaSuccess)
        return err;
    for (int variant : {(int) kVariantPlain, (int) kVariantPred, (int) kVariantPriv, (int) kVariantLook, (int) kVariantLook64, (int) kVariantLook1,
                        (int) kVariantLookRing1})
        for (bool uniform : {false, true})
            for (bool starts : {false, true}) {
                const void* fn = BatchKernelFor(variant, uniform, starts).fn;
                err = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, optin);
                if (err != cudaSuccess)
                    return err;
                // three CTAs of ~75 KB each per SM: ask for the largest shared-memory carve-out (kernels without a
                // blocks-per-SM launch bound would otherwise get a smaller one and run two CTAs)
                err = cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
                if (err != cudaSuccess)
                    return err;
            }
    return cudaSuccess;
}

cudaError_t PlanScan(int device, uint32_t hot, uint32_t hot_small, uint32_t priv_rows, int variant, bool uniform, LaunchPlan* plan,
                     bool starts)
{
    const BatchKernel k = BatchKernelFor(variant, uniform, starts);
    const bool priv = variant == kVariantPriv && uniform && !starts;
    plan->block = k.block;
    plan->shared = priv ? ScanSharedBytes(hot_small, priv_rows) : uniform ? ScanSharedBytes(hot, 0) : GenericSharedBytes(hot);
    plan->shared += (size_t) (plan->block / 32) * k.ring_warp_bytes;         // every warp's ring after the tables
    int sms = 0, per_sm = 0;
    cudaError_t err = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (err != cudaSuccess)
        return err;
    err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k.fn, plan->block, plan->shared);
    if (err != cudaSuccess)
        return err;
    if (per_sm < 1)
        return cudaErrorLaunchOutOfResources;
    if (!uniform)
        per_sm = per_sm < kGenericBlocksPerSM ? per_sm : kGenericBlocksPerSM;      // a third CTA measured slower twice (r01, r02 notes)
    plan->grid = sms * per_sm;     // persistent: every SM holds its full share of CTAs
    return cudaSuccess;
}

cudaError_t LaunchScan(const ScanArgs& a, int variant, bool uniform, const LaunchPlan& plan, cudaStream_t stream)
{
    if (a.n == 0)
        return cudaSuccess;
    const BatchKernel k = BatchKernelFor(variant, uniform, a.starts != nullptr);
    const uint64_t units = ((a.n + 31) / 32 + k.units_per_step - 1) / k.units_per_step;
    const uint64_t warps_per_block = (uint64_t) plan.block / 32;
    uint64_t want = (units + warps_per_block - 1) / warps_per_block;
    int grid = (int) (want < (uint64_t) plan.grid ? want : (uint64_t) plan.grid);
    void* args[] = {const_cast<ScanArgs*>(&a)};
    cudaError_t err = cudaLaunchKernel(k.fn, dim3(grid), dim3(plan.block), args, plan.shared, stream);
    if (err == cudaSuccess)
        g_launches.fetch_add(1, std::memory_order_relaxed);
    return err;
}

// Length-ordered CSR batch: the leading long strings, one per warp (ScanSplitKernel).  a.split_count / a.split_counter
// are two device words; the generic kernel launched afterwards with the same a.split_count skips those strings.
cudaError_t LaunchSplit(const ScanArgs& a, int variant, int device, cudaStream_t stream)
{
    if (a.n == 0)
        return cudaSuccess;
    SplitCountKernel<<<1, 32, 0, stream>>>(a.offsets, a.order, a.n, kSplitMin, const_cast<uint32_t*>(a.split_count), a.split_counter);
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess)
        return err;
    g_launches.fetch_add(1, std::memory_order_relaxed);
    static const uint32_t split_prefetch = [] {
        const char* env = getenv("PIRE_B200_SPLIT_PREFETCH");     // blocks of 32 bytes between the walk and its L2 prefetch; 0 = none
        return env ? (uint32_t) atoi(env) : 0u;
    }();
    const void* fn = a.starts ? (variant == kVariantPlain ? reinterpret_cast<const void*>(&ScanSplitKernel<false, true>)
                                                          : reinterpret_cast<const void*>(&ScanSplitKernel<true, true>))
                              : (variant == kVariantPlain ? reinterpret_cast<const void*>(&ScanSplitKernel<false, false>)
                                                          : reinterpret_cast<const void*>(&ScanSplitKernel<true, false>));
    const size_t shared = ScanSharedBytes(a.hot, 0) + kSplitMarkBytes + kWarpsPerBlock * 32;
    int optin = 0, sms = 0, per_sm = 0;
    err = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    if (err == cudaSuccess)
        err = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (err == cudaSuccess)
        err = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, optin);
    if (err == cudaSuccess)
        err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kBlock, shared);
    if (err != cudaSuccess)
        return err;
    if (per_sm < 1)
        return cudaErrorLaunchOutOfResources;
    ScanArgs with_prefetch = a;                 // kernel arguments are copied at launch
    with_prefetch.split_prefetch = split_prefetch;
    void* args[] = {&with_prefetch};
    err = cudaLaunchKernel(fn, dim3(sms * per_sm), dim3(kBlock), args, shared, stream);
    if (err == cudaSuccess)
        g_launches.fetch_add(1, std::memory_order_relaxed);
    return err;
}

// One string (a.corpus, a.fixed_len bytes) over the persistent grid (ScanStringKernel, CountStringKernel).  The grid is the occupancy
// query's, cut to one CTA per kBlock * kStringMinBlocks blocks of body so that pieces do not get short; every length,
// down to 0, goes through the kernel.  a.string_ends / a.string_rounds (and with `sums`, a.string_sums) are filled in
// here from per-call scratch.
static cudaError_t LaunchStringGrid(const void* fn, const ScanArgs& a, size_t shared, int device, cudaStream_t stream,
                                    bool sums = false)
{
    int optin = 0, sms = 0, per_sm = 0;
    cudaError_t err = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    if (err == cudaSuccess)
        err = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (err == cudaSuccess)
        err = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, optin);
    if (err == cudaSuccess)
        err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kBlock, shared);
    if (err != cudaSuccess)
        return err;
    if (per_sm < 1)
        return cudaErrorLaunchOutOfResources;
    const uint64_t blocks = a.fixed_len / 32;
    const uint64_t want = (blocks + (uint64_t) kBlock * kStringMinBlocks - 1) / ((uint64_t) kBlock * kStringMinBlocks);
    const uint64_t full = (uint64_t) sms * (uint64_t) per_sm;
    const int grid = (int) (want < 1 ? 1 : want < full ? want : full);
    // rounds counters (3 words), then the warps' ends, double-buffered, then (sums) one u64 per CTA
    uint32_t* scratch = nullptr;
    const size_t words = 4 + 2 * (size_t) grid * kWarpsPerBlock + (sums ? 2 * (size_t) grid : 0);
    err = ScratchAlloc(reinterpret_cast<void**>(&scratch), words * 4, stream);
    if (err != cudaSuccess)
        return err;
    err = cudaMemsetAsync(scratch, 0, 4 * 4, stream);
    ScanArgs with_scratch = a;
    with_scratch.string_rounds = scratch;
    with_scratch.string_ends = scratch + 4;
    if (sums)
        with_scratch.string_sums = reinterpret_cast<unsigned long long*>(scratch + 4 + 2 * (size_t) grid * kWarpsPerBlock);
    void* args[] = {&with_scratch};
    if (err == cudaSuccess)
        err = cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(kBlock), args, shared, stream);
    if (err == cudaSuccess)
        g_launches.fetch_add(1, std::memory_order_relaxed);
    cudaFreeAsync(scratch, stream);
    return err;
}

cudaError_t LaunchString(const ScanArgs& a, int variant, int device, cudaStream_t stream)
{
    const void* fn = variant == kVariantPlain ? reinterpret_cast<const void*>(&ScanStringKernel<false>)
                                              : reinterpret_cast<const void*>(&ScanStringKernel<true>);
    return LaunchStringGrid(fn, a, ScanSharedBytes(a.hot, 0) + kSplitMarkBytes, device, stream);
}

// Behind the tables and the marks: the hot states' packed increments, then (a.count_rows) one row of u32 per warp.
cudaError_t LaunchCountString(const ScanArgs& a, int device, cudaStream_t stream)
{
    const void* fn = nullptr;
    switch (a.count_words * 2 + (a.count_always ? 1 : 0)) {
    case 2: fn = reinterpret_cast<const void*>(&CountStringKernel<1, false>); break;
    case 3: fn = reinterpret_cast<const void*>(&CountStringKernel<1, true>); break;
    case 4: fn = reinterpret_cast<const void*>(&CountStringKernel<2, false>); break;
    case 5: fn = reinterpret_cast<const void*>(&CountStringKernel<2, true>); break;
    default: fn = reinterpret_cast<const void*>(&CountStringKernel<0, false>); break;
    }
    const size_t shared = ScanSharedBytes(a.hot, 0) + kSplitMarkBytes + (size_t) (a.hot + 1) * a.count_words * 8
                          + (a.count_rows ? (size_t) kWarpsPerBlock * a.regexps * 4 : 0);
    return LaunchStringGrid(fn, a, shared, device, stream);
}

// Behind the tables and the marks: the scan's words (kWarpsPerBlock + 2 u64), then the hot states' list lengths.
cudaError_t LaunchMatchEndsString(const ScanArgs& a, int device, cudaStream_t stream)
{
    const size_t shared = ScanSharedBytes(a.hot, 0) + kSplitMarkBytes + (kWarpsPerBlock + 2) * 8 + (size_t) a.hot * 4;
    return LaunchStringGrid(reinterpret_cast<const void*>(&MatchEndsStringKernel), a, shared, device, stream, true);
}

cudaError_t LaunchPrefix(const ScanArgs& a, bool shortest, bool reverse, int device, cudaStream_t stream)
{
    if (a.n == 0)
        return cudaSuccess;
    const void* fn = reverse ? (shortest ? reinterpret_cast<const void*>(&PrefixKernel<true, true>)
                                         : reinterpret_cast<const void*>(&PrefixKernel<false, true>))
                             : (shortest ? reinterpret_cast<const void*>(&PrefixKernel<true, false>)
                                         : reinterpret_cast<const void*>(&PrefixKernel<false, false>));
    int optin = 0, sms = 0;
    cudaError_t err = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    if (err == cudaSuccess)
        err = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (err == cudaSuccess)
        err = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, optin);
    if (err != cudaSuccess)
        return err;
    if (a.uniform && !reverse) {
        const int block = 640;                                         // two CTAs of twenty warps at 48 registers
        fn = shortest ? reinterpret_cast<const void*>(&PrefixUniformKernel<true>) : reinterpret_cast<const void*>(&PrefixUniformKernel<false>);
        const size_t shared = ScanSharedBytes(a.hot, 0) + 272;
        int per_sm = 0;
        err = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, optin);
        if (err == cudaSuccess)
            err = cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        if (err == cudaSuccess)
            err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, block, shared);
        if (err != cudaSuccess)
            return err;
        if (per_sm < 1)
            return cudaErrorLaunchOutOfResources;
        const uint64_t per_block = (uint64_t) block;
        const uint64_t want = (a.n + per_block - 1) / per_block;
        const int grid = (int) (want < (uint64_t) sms * per_sm ? want : (uint64_t) sms * per_sm);
        void* args[] = {const_cast<ScanArgs*>(&a)};
        err = cudaLaunchKernel(fn, dim3(grid), dim3(block), args, shared, stream);
        if (err == cudaSuccess)
            g_launches.fetch_add(1, std::memory_order_relaxed);
        return err;
    }
    const size_t shared = GenericSharedBytes(a.hot) + 272;      // + the hot states' flag bytes
    uint64_t want = (a.n + kBlock - 1) / kBlock;
    int grid = (int) (want < (uint64_t) sms * kGenericBlocksPerSM ? want : (uint64_t) sms * kGenericBlocksPerSM);
    void* args[] = {const_cast<ScanArgs*>(&a)};
    err = cudaLaunchKernel(fn, dim3(grid), dim3(kBlock), args, shared, stream);
    if (err == cudaSuccess)
        g_launches.fetch_add(1, std::memory_order_relaxed);
    return err;
}


// Lines of text (CSR, PIRE_GPU_RUN_LINES, no order).  The caller zeroes the bitmap.  In stream (ScanTextKernel) when the
// start state is a hot row -- it practically always is; lanes pulling lines one by one (ScanLinesKernel) otherwise.
cudaError_t LaunchLines(const ScanArgs& a, int variant, int device, cudaStream_t stream)
{
    if (a.n == 0)
        return cudaSuccess;
    const bool in_stream = a.start < a.hot;
    const bool pred = WalkMode(variant) != 0;
    const void* fn = in_stream ? (pred ? reinterpret_cast<const void*>(&ScanTextKernel<true>) : reinterpret_cast<const void*>(&ScanTextKernel<false>))
                               : (pred ? reinterpret_cast<const void*>(&ScanLinesKernel<true>) : reinterpret_cast<const void*>(&ScanLinesKernel<false>));
    const size_t shared = ScanSharedBytes(a.hot, 0) + (in_stream ? kTextFinBytes + kTextPackBytes : 0);
    int optin = 0, sms = 0, per_sm = 0;
    cudaError_t err = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    if (err == cudaSuccess)
        err = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (err == cudaSuccess)
        err = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, optin);
    if (err == cudaSuccess)
        err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kBlock, shared);
    if (err != cudaSuccess)
        return err;
    if (per_sm < 1)
        return cudaErrorLaunchOutOfResources;
    ScanArgs tuned = a;
    int grid = sms * per_sm;
    // in stream, the persistent grid is launched whole: the number of units depends on the text's size, which only the
    // device knows (offsets[n]); warps without a unit leave at once
    if (!in_stream) {
        const uint64_t groups = (a.n + kLinesPerWarp - 1) / kLinesPerWarp;
        const uint64_t want = (groups + kWarpsPerBlock - 1) / kWarpsPerBlock;
        grid = (int) (want < (uint64_t) grid ? want : (uint64_t) grid);
        tuned.lines_turn = kPiecesPerTurn;
        tuned.lines_min_idle = kLinesMinIdle;
    }
    void* args[] = {&tuned};
    err = cudaLaunchKernel(fn, dim3(grid), dim3(kBlock), args, shared, stream);
    if (err == cudaSuccess)
        g_launches.fetch_add(1, std::memory_order_relaxed);
    return err;
}

template <bool kFrom>
static const void* CountKernelFor(const ScanArgs& a)
{
    switch (a.count_words * 2 + (a.count_always ? 1 : 0)) {
    case 2: return reinterpret_cast<const void*>(&CountKernel<1, false, kFrom>);
    case 3: return reinterpret_cast<const void*>(&CountKernel<1, true, kFrom>);
    case 4: return reinterpret_cast<const void*>(&CountKernel<2, false, kFrom>);
    case 5: return reinterpret_cast<const void*>(&CountKernel<2, true, kFrom>);
    default: return reinterpret_cast<const void*>(&CountKernel<0, false, kFrom>);
    }
}

cudaError_t LaunchCount(const ScanArgs& a, int device, cudaStream_t stream, bool from)
{
    if (a.n == 0)
        return cudaSuccess;
    const void* fn = from ? CountKernelFor<true>(a) : CountKernelFor<false>(a);
    int optin = 0, sms = 0;
    cudaError_t err = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    if (err == cudaSuccess)
        err = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (err == cudaSuccess)
        err = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, optin);
    if (err != cudaSuccess)
        return err;
    const size_t shared = GenericSharedBytes(a.hot) + (size_t) (a.hot + 1) * a.count_words * 8;
    const uint64_t want = ((a.n + 31) / 32 + kWarpsPerBlock - 1) / kWarpsPerBlock;
    int grid = (int) (want < (uint64_t) sms * kGenericBlocksPerSM ? want : (uint64_t) sms * kGenericBlocksPerSM);
    void* args[] = {const_cast<ScanArgs*>(&a)};
    err = cudaLaunchKernel(fn, dim3(grid), dim3(kBlock), args, shared, stream);
    if (err == cudaSuccess)
        g_launches.fetch_add(1, std::memory_order_relaxed);
    return err;
}

// Two walks of CountKernel's shape around a scan.  The counting walk leaves n + 1 words [*a.found, entries of string 0,
// ..., entries of string n - 1] and the strings' last states in scratch; their inclusive sum (cub::DeviceScan) is where
// each string's slice begins, and its last word the new *a.found; the writing walk places every string's entries there.
// The arrays are thus the same on every run, and a short buffer holds exactly the answer's first a.ends_capacity entries.
cudaError_t LaunchMatchEndsBatch(const ScanArgs& a, int device, cudaStream_t stream)
{
    if (a.n == 0)
        return cudaSuccess;
    const void* count = reinterpret_cast<const void*>(&MatchEndsBatchKernel<false>);
    const void* emit = reinterpret_cast<const void*>(&MatchEndsBatchKernel<true>);
    int optin = 0, sms = 0;
    cudaError_t err = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    if (err == cudaSuccess)
        err = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (err == cudaSuccess)
        err = cudaFuncSetAttribute(count, cudaFuncAttributeMaxDynamicSharedMemorySize, optin);
    if (err == cudaSuccess)
        err = cudaFuncSetAttribute(emit, cudaFuncAttributeMaxDynamicSharedMemorySize, optin);
    if (err != cudaSuccess)
        return err;
    const uint64_t items = a.n + 1;
    unsigned long long *counts = nullptr, *first = nullptr;
    uint32_t* last = nullptr;
    void* temp = nullptr;
    size_t temp_bytes = 0;
    err = cub::DeviceScan::InclusiveSum(nullptr, temp_bytes, counts, first, items, stream);
    if (err == cudaSuccess) err = ScratchAlloc(reinterpret_cast<void**>(&counts), items * 8, stream);
    if (err == cudaSuccess) err = ScratchAlloc(reinterpret_cast<void**>(&first), items * 8, stream);
    if (err == cudaSuccess) err = ScratchAlloc(reinterpret_cast<void**>(&last), a.n * 4, stream);
    if (err == cudaSuccess) err = ScratchAlloc(&temp, temp_bytes, stream);
    const uint64_t want = ((a.n + 31) / 32 + kWarpsPerBlock - 1) / kWarpsPerBlock;
    const int grid = (int) (want < (uint64_t) sms * kGenericBlocksPerSM ? want : (uint64_t) sms * kGenericBlocksPerSM);
    ScanArgs walk = a;
    walk.ends_base = 0;
    walk.entry_counts = counts;
    walk.entry_first = first;
    walk.last_states = last;
    void* args[] = {&walk};
    if (err == cudaSuccess) {
        // behind the staging ring: the hot states' list lengths (the writing walk leaves them unused)
        err = cudaLaunchKernel(count, dim3(grid), dim3(kBlock), args, GenericSharedBytes(a.hot) + (size_t) a.hot * 4, stream);
        if (err == cudaSuccess)
            g_launches.fetch_add(1, std::memory_order_relaxed);
    }
    if (err == cudaSuccess)
        err = cub::DeviceScan::InclusiveSum(temp, temp_bytes, counts, first, items, stream);
    if (err == cudaSuccess) {
        err = cudaLaunchKernel(emit, dim3(grid), dim3(kBlock), args, GenericSharedBytes(a.hot), stream);
        if (err == cudaSuccess)
            g_launches.fetch_add(1, std::memory_order_relaxed);
    }
    if (counts) cudaFreeAsync(counts, stream);
    if (first) cudaFreeAsync(first, stream);
    if (last) cudaFreeAsync(last, stream);
    if (temp) cudaFreeAsync(temp, stream);
    return err;
}

cudaError_t LaunchVisitCount(const ScanArgs& a, cudaStream_t stream)
{
    if (a.n == 0)
        return cudaSuccess;
    int grid = (int) ((a.n + 255) / 256);
    VisitCountKernel<<<grid, 256, 0, stream>>>(a);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}

namespace {
__global__ void __launch_bounds__(256) LengthKeysKernel(const uint64_t* __restrict__ offsets, uint64_t n, uint32_t* __restrict__ keys,
                                                        uint32_t* __restrict__ ids)
{
    const uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        // Bucket = half an octave of length.  The sort is stable and only on the bucket, so
        // inside a bucket strings keep their corpus order: the 32 lanes of a warp then read
        // from neighbouring addresses (a full sort by length scatters them over the whole
        // corpus, which measured 4x slower than the imbalance it removes -- r01 experiments).
        uint64_t len = offsets[i + 1] - offsets[i];
        uint32_t l32 = (uint32_t) (len > 0xffffffffull ? 0xffffffffull : len);
        uint32_t msb = l32 ? 31u - (uint32_t) __clz(l32) : 0u;
        uint32_t half = msb ? (l32 >> (msb - 1)) & 1u : 0u;
        keys[i] = 255u - (msb * 2u + half);                                     // ascending keys = longest bucket first
        ids[i] = (uint32_t) i;
    }
}
} // namespace

// Stream-ordered scratch (work counters, sort/select temporaries) comes from a private per-device pool
// that keeps up to 64 MiB cached.  The device's default pool returns everything to the driver at each
// synchronisation, after which the next 4-byte counter allocation costs a 10-40 ms mapping stall -- seen as
// one slow step in twenty on the length-binned path.
// A persistent grid of the generic kernel's shape; behind the staging ring: the hot states' flag bytes (272), accept
// masks (256 words) and, up to kStartsHotLiveWords words a row, their live rows.
cudaError_t LaunchMatchStarts(const ScanArgs& a, int device, cudaStream_t stream)
{
    const void* fn = reinterpret_cast<const void*>(&MatchStartsKernel);
    int optin = 0, sms = 0;
    cudaError_t err = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    if (err == cudaSuccess)
        err = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (err == cudaSuccess)
        err = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, optin);
    if (err != cudaSuccess)
        return err;
    const size_t shared = GenericSharedBytes(a.hot) + 272 + 256 * 4
                          + (a.live_words <= kStartsHotLiveWords ? (size_t) a.hot * a.live_words * 4 : 0);
    ScanArgs walk = a;
    err = ScratchAlloc(reinterpret_cast<void**>(&walk.group_counter), 8, stream);
    if (err != cudaSuccess)
        return err;
    err = cudaMemsetAsync(walk.group_counter, 0, 8, stream);
    if (err == cudaSuccess) {
        void* args[] = {&walk};
        err = cudaLaunchKernel(fn, dim3(sms * kGenericBlocksPerSM), dim3(kBlock), args, shared, stream);
        if (err == cudaSuccess)
            g_launches.fetch_add(1, std::memory_order_relaxed);
    }
    cudaFreeAsync(walk.group_counter, stream);
    return err;
}

cudaError_t ScratchAlloc(void** out, size_t bytes, cudaStream_t stream)
{
    static std::mutex mu;
    static cudaMemPool_t pools[64] = {};
    int device = 0;
    cudaError_t err = cudaGetDevice(&device);
    if (err != cudaSuccess)
        return err;
    if (device < 0 || device >= 64)
        return cudaMallocAsync(out, bytes, stream);
    cudaMemPool_t pool;
    {
        std::lock_guard<std::mutex> lock(mu);
        if (!pools[device]) {
            cudaMemPoolProps props = {};
            props.allocType = cudaMemAllocationTypePinned;
            props.handleTypes = cudaMemHandleTypeNone;
            props.location.type = cudaMemLocationTypeDevice;
            props.location.id = device;
            err = cudaMemPoolCreate(&pools[device], &props);
            if (err != cudaSuccess)
                return err;
            uint64_t keep = 64ull << 20;
            err = cudaMemPoolSetAttribute(pools[device], cudaMemPoolAttrReleaseThreshold, &keep);
            if (err != cudaSuccess)
                return err;
        }
        pool = pools[device];
    }
    return cudaMallocFromPoolAsync(out, bytes, pool, stream);
}

cudaError_t LengthOrder(const uint64_t* d_offsets, uint64_t n, uint32_t* d_order, cudaStream_t stream)
{
    if (n == 0)
        return cudaSuccess;
    uint32_t *keys = nullptr, *keys_out = nullptr, *ids = nullptr;
    void* temp = nullptr;
    size_t temp_bytes = 0;
    cudaError_t err = ScratchAlloc((void**) &keys, n * 4, stream);
    if (err == cudaSuccess) err = ScratchAlloc((void**) &keys_out, n * 4, stream);
    if (err == cudaSuccess) err = ScratchAlloc((void**) &ids, n * 4, stream);
    if (err == cudaSuccess) {
        LengthKeysKernel<<<(unsigned) ((n + 255) / 256), 256, 0, stream>>>(d_offsets, n, keys, ids);
        g_launches.fetch_add(1, std::memory_order_relaxed);
        err = cudaGetLastError();
    }
    if (err == cudaSuccess)
        err = cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, keys, keys_out, ids, d_order, (int) n, 0, 8, stream);
    if (err == cudaSuccess) err = ScratchAlloc(&temp, temp_bytes, stream);
    if (err == cudaSuccess)
        err = cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys, keys_out, ids, d_order, (int) n, 0, 8, stream);
    if (keys) cudaFreeAsync(keys, stream);
    if (keys_out) cudaFreeAsync(keys_out, stream);
    if (ids) cudaFreeAsync(ids, stream);
    if (temp) cudaFreeAsync(temp, stream);
    return err;
}

namespace {
struct IsNewline {
    const uint8_t* text;
    __host__ __device__ bool operator()(const unsigned long long& i) const { return text[i] == '\n'; }
};

__global__ void __launch_bounds__(256) CountNewlinesKernel(const uint8_t* __restrict__ text, uint64_t n_bytes, unsigned long long* __restrict__ count)
{
    unsigned long long local = 0;
    for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n_bytes; i += (uint64_t) gridDim.x * blockDim.x)
        local += text[i] == '\n';
    for (int d = 16; d; d >>= 1)
        local += __shfl_down_sync(0xffffffffu, local, d);
    if ((threadIdx.x & 31) == 0 && local)
        atomicAdd(count, local);
}

__global__ void FinishLineOffsetsKernel(const uint8_t* __restrict__ text, uint64_t n_bytes, uint64_t* __restrict__ offsets,
                                        const unsigned long long* __restrict__ n_newlines, uint64_t capacity,
                                        unsigned long long* __restrict__ n_lines_out)
{
    // offsets[1..k] hold newline positions; turn them into the starts of the following lines
    const unsigned long long k = *n_newlines;
    const uint64_t idx = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < k && idx + 1 <= capacity)
        offsets[idx + 1] += 1;
    if (idx == 0) {
        offsets[0] = 0;
        unsigned long long lines = k;
        if (n_bytes != 0 && text[n_bytes - 1] != '\n') {     // last line has no newline: a virtual one after the end
            if (k + 1 <= capacity)
                offsets[k + 1] = n_bytes + 1;
            lines = k + 1;
        }
        *n_lines_out = lines;
    }
}
} // namespace

cudaError_t SplitLines(const uint8_t* d_text, uint64_t n_bytes, uint64_t* d_offsets, uint64_t capacity, uint64_t* n_lines,
                       cudaStream_t stream)
{
    *n_lines = 0;
    if (n_bytes == 0)
        return cudaSuccess;
    unsigned long long* d_counts = nullptr;       // [0] newlines, [1] lines
    void* temp = nullptr;
    size_t temp_bytes = 0;
    cudaError_t err = ScratchAlloc((void**) &d_counts, 2 * sizeof(unsigned long long), stream);
    cub::CountingInputIterator<unsigned long long> positions(0);
    IsNewline pred{d_text};
    unsigned long long* out = reinterpret_cast<unsigned long long*>(d_offsets + 1);
    // capacity guards: the select writes at most min(newlines, n_bytes) entries; the caller sizes d_offsets for the
    // worst case it accepts (capacity + 1 entries) and we verify after the fact.
    // first pass: how many lines?  (the select below writes every newline position, so the
    // caller's buffer must be known to be large enough before it runs)
    unsigned long long precount = 0;
    if (err == cudaSuccess)
        err = cudaMemsetAsync(d_counts, 0, 2 * sizeof(unsigned long long), stream);
    if (err == cudaSuccess) {
        uint64_t blocks = (n_bytes + 256 * 64 - 1) / (256 * 64);
        CountNewlinesKernel<<<(unsigned) (blocks < GridCap(16) ? blocks : GridCap(16)), 256, 0, stream>>>(d_text, n_bytes, d_counts);
        g_launches.fetch_add(1, std::memory_order_relaxed);
        err = cudaGetLastError();
    }
    if (err == cudaSuccess)
        err = cudaMemcpyAsync(&precount, d_counts, sizeof(precount), cudaMemcpyDeviceToHost, stream);
    if (err == cudaSuccess)
        err = cudaStreamSynchronize(stream);
    if (err == cudaSuccess && (!d_offsets || precount + 1 > capacity)) {
        cudaFreeAsync(d_counts, stream);
        *n_lines = precount + 1;                       // upper bound of lines; caller retries with this capacity
        return cudaErrorInvalidValue;
    }
    if (err == cudaSuccess)
        err = cub::DeviceSelect::If(nullptr, temp_bytes, positions, out, d_counts, (long long) n_bytes, pred, stream);
    if (err == cudaSuccess)
        err = ScratchAlloc(&temp, temp_bytes, stream);
    if (err == cudaSuccess)
        err = cub::DeviceSelect::If(temp, temp_bytes, positions, out, d_counts, (long long) n_bytes, pred, stream);
    unsigned long long newlines = 0;
    if (err == cudaSuccess)
        err = cudaMemcpyAsync(&newlines, d_counts, sizeof(newlines), cudaMemcpyDeviceToHost, stream);
    if (err == cudaSuccess)
        err = cudaStreamSynchronize(stream);
    if (err == cudaSuccess) {
        unsigned blocks = (unsigned) ((newlines + 255) / 256);
        FinishLineOffsetsKernel<<<blocks ? blocks : 1, 256, 0, stream>>>(d_text, n_bytes, d_offsets, d_counts, capacity, d_counts + 1);
        g_launches.fetch_add(2, std::memory_order_relaxed);
        err = cudaGetLastError();
    }
    unsigned long long lines = 0;
    if (err == cudaSuccess)
        err = cudaMemcpyAsync(&lines, d_counts + 1, sizeof(lines), cudaMemcpyDeviceToHost, stream);
    if (err == cudaSuccess)
        err = cudaStreamSynchronize(stream);
    if (d_counts) cudaFreeAsync(d_counts, stream);
    if (temp) cudaFreeAsync(temp, stream);
    *n_lines = lines;
    return err;
}

cudaError_t LaunchSynth(const SynthParams& p, const char* d_plants, uint8_t* d_out, cudaStream_t stream)
{
    if (p.n_strings == 0)
        return cudaSuccess;
    uint64_t total = p.n_strings * (p.string_len / 16);
    uint64_t blocks = (total + 255) / 256;
    int grid = (int) (blocks < GridCap(64) ? blocks : GridCap(64));
    SynthKernel<<<grid, 256, 0, stream>>>(p, d_plants, d_out);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}

cudaError_t LaunchSynthMixedLengths(uint64_t seed, uint64_t first, uint64_t n, uint64_t* d_lengths, cudaStream_t stream)
{
    if (n == 0)
        return cudaSuccess;
    SynthMixedLengthsKernel<<<(unsigned) ((n + 255) / 256), 256, 0, stream>>>(seed, first, n, d_lengths);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}

cudaError_t LaunchSynthMixedFill(uint64_t seed, uint32_t plant_every, uint64_t first, uint64_t n, const uint64_t* d_offsets,
                                 uint8_t* d_out, cudaStream_t stream)
{
    if (n == 0)
        return cudaSuccess;
    uint64_t blocks = (n + 7) / 8;
    SynthMixedFillKernel<<<(unsigned) (blocks < GridCap(32) ? blocks : GridCap(32)), 256, 0, stream>>>(seed, plant_every, first, n,
                                                                                                   d_offsets, d_out);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}

namespace {
// AcceptedRegexps of the state every string stopped in, as a bit set of `words` 32-bit words (multi.h:149-158 for
// scanners with more than 32 regexps; the scan kernels' accept mask holds ids 0..31 only).
__global__ void __launch_bounds__(256) AcceptGatherKernel(const uint32_t* __restrict__ table, uint32_t states, uint32_t words,
                                                          const uint32_t* __restrict__ state_idx, uint64_t n, uint32_t* __restrict__ out)
{
    const uint64_t total = n * words;
    for (uint64_t k = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (uint64_t) gridDim.x * blockDim.x) {
        const uint64_t i = k / words;
        const uint32_t w = (uint32_t) (k % words);
        const uint32_t st = state_idx[i];
        out[k] = st < states ? __ldg(table + (size_t) st * words + w) : 0u;
    }
}
} // namespace

cudaError_t LaunchAcceptGather(const uint32_t* d_table, uint32_t states, uint32_t words, const uint32_t* d_state_idx, uint64_t n,
                               uint32_t* d_out, cudaStream_t stream)
{
    if (n == 0 || words == 0)
        return cudaSuccess;
    const uint64_t total = n * words;
    const uint64_t blocks = (total + 255) / 256;
    AcceptGatherKernel<<<(unsigned) (blocks < GridCap(32) ? blocks : GridCap(32)), 256, 0, stream>>>(d_table, states, words, d_state_idx, n, d_out);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}

uint64_t KernelLaunchCount() { return g_launches.load(std::memory_order_relaxed); }

} // namespace pire_b200
