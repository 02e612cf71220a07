// tools/microbench.cu -- how fast can one-string-per-lane loads pull a corpus of
// 1 KiB strings out of HBM?  Measures the load path of the scan kernel in
// isolation (XOR-reduce, no table walk) for several load shapes, so that the
// scan kernel's distance from the HBM roofline can be attributed to the walk
// (shared-memory wavefronts) or to the loads (L1TEX tag stage: 32 distinct
// lines per warp-wide request).  Not part of the product library.
//
// The "flagship" rows run at the glued scan's shapes: the register kernel's residency (two CTAs of 448 threads, 28
// warps per SM) with two strings per lane (units 2p and 2p+1 of a pair, one 32-byte block of each in flight), and a
// TMA-staged alternative (one CTA of 1024 threads per SM, a per-warp ring of 64-row x 32-byte tiles read with
// LDS.128), the shape a shared-memory-fed walk would need beside a 75 KB hot table.  The "ring" rows feed the same two
// strings per lane from a per-lane cp.async ring in shared memory (one CTA per SM beside 76 KB held back for the table),
// the input side of ScanUniformLookRingKernel, at several (warps, slots) shapes, .ca / .cg and L2 prefetch-size hints.
//
// The "ring1" rows keep one string per lane in the same kind of ring, the input side of ScanUniformLookRing1Kernel.
//
//   microbench [GiB=4] [string_len=1024] [ring]     ("ring": only the ring comparison rows; any other third argument:
//                                                    only the pipe rows)
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#define CK(x)                                                                                   \
    do {                                                                                        \
        cudaError_t e__ = (x);                                                                  \
        if (e__ != cudaSuccess) {                                                               \
            std::fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e__)); \
            std::exit(1);                                                                       \
        }                                                                                       \
    } while (0)

__device__ __forceinline__ uint4 Ld16(const uint8_t* p)
{
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ uint4 Ld16Alloc(const uint8_t* p)
{
    uint4 v;
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
// sm_90 has no 256-bit load: 32 bytes of a lane are two 128-bit loads of one sector.  kL1: whether they allocate in
// L1 (then the second half of the sector is an L1 hit; without, both halves go to L2).  The first load carries the
// 256-byte L2 prefetch hint.
template <bool kL1>
__device__ __forceinline__ void Ld32(const uint8_t* p, uint4& a, uint4& b)
{
    if (kL1)
        asm volatile("ld.global.nc.L2::256B.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
                     "ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                     : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w), "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w)
                     : "l"(p));
    else
        asm volatile("ld.global.nc.L1::no_allocate.L2::256B.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
                     "ld.global.nc.L1::no_allocate.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                     : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w), "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w)
                     : "l"(p));
}
__device__ __forceinline__ uint32_t Fold(uint4 v) { return v.x ^ v.y ^ v.z ^ v.w; }

// The load of the register-fed uniform kernels (ScanUniformKernel, ScanUniformLookKernel): two LDG.128 of one sector,
// both allocating in L1.  kL2 = 0, 64, 128 or 256: the first load carries the L2 prefetch-size hint of that many bytes.
template <int kL2>
__device__ __forceinline__ void Ld32Pair(const uint8_t* p, uint4& a, uint4& b)
{
    if (kL2 == 64)
        asm volatile("ld.global.nc.L2::64B.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
                     "ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                     : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w), "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w) : "l"(p));
    else if (kL2 == 128)
        asm volatile("ld.global.nc.L2::128B.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
                     "ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                     : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w), "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w) : "l"(p));
    else if (kL2 == 256)
        asm volatile("ld.global.nc.L2::256B.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
                     "ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                     : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w), "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w) : "l"(p));
    else
        asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
                     "ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                     : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w), "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w) : "l"(p));
}

// Two strings per lane (rows 64p + lane and 64p + 32 + lane), the next 32-byte block of both in flight while the
// current one is folded: the input side of the register-fed two-string look-ahead kernel (ScanUniformLook2Kernel, since
// removed; the ring kernel replaced it) without the walk.
template <int kL2>
__global__ void __launch_bounds__(448) LoadPairKernel(const uint8_t* corpus, uint64_t n, uint32_t len, uint32_t* out)
{
    const uint64_t warps = (uint64_t) gridDim.x * (blockDim.x / 32);
    const uint32_t lane = threadIdx.x & 31;
    uint32_t acc = 0;
    for (uint64_t pair = (uint64_t) blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); pair < n / 64; pair += warps) {
        const uint8_t* pa = corpus + (pair * 64 + lane) * (uint64_t) len;
        const uint8_t* pb = pa + 32 * (uint64_t) len;
        uint4 a0, a1, b0, b1, c0, c1, d0, d1;
        Ld32Pair<kL2>(pa, a0, a1);
        Ld32Pair<kL2>(pb, b0, b1);
        for (uint32_t off = 32; off < len; off += 32) {
            Ld32Pair<kL2>(pa + off, c0, c1);
            Ld32Pair<kL2>(pb + off, d0, d1);
            acc ^= Fold(a0) ^ Fold(a1) ^ Fold(b0) ^ Fold(b1);
            a0 = c0; a1 = c1; b0 = d0; b1 = d1;
        }
        acc ^= Fold(a0) ^ Fold(a1) ^ Fold(b0) ^ Fold(b1);
    }
    if (acc == 0x12345678u)
        out[0] = acc;
}

// ---- TMA tiles: one CTA of 32 warps per SM, each warp a ring of kStages tiles of 64 rows x 32 bytes (SWIZZLE_32B)
constexpr uint32_t kTileBytes = 64 * 32;

__device__ __forceinline__ void MbarWait(uint32_t bar, uint32_t parity)
{
    asm volatile("{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@!p bra W_%=;\n}\n" ::"r"(bar),
                 "r"(parity) : "memory");
}

__device__ __forceinline__ void IssueTile(uint32_t dst, uint32_t bar, const CUtensorMap* tm, uint32_t x, uint32_t y)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "n"(kTileBytes) : "memory");
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
                 "l"(tm), "r"(x), "r"(y), "r"(bar)
                 : "memory");
}

template <int kStages>
__global__ void __launch_bounds__(1024, 1) TmaTileKernel(const __grid_constant__ CUtensorMap tm, uint64_t n, uint32_t len, uint32_t* out)
{
    extern __shared__ __align__(1024) uint8_t tiles[];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t warps = gridDim.x * (blockDim.x / 32);
    const uint32_t ring = (uint32_t) __cvta_generic_to_shared(tiles) + warp * kStages * kTileBytes;
    const uint32_t bars = (uint32_t) __cvta_generic_to_shared(tiles) + 32 * kStages * kTileBytes + warp * kStages * 8;
    if (ring & 1023)
        __trap();
    if (lane == 0) {
        for (int s = 0; s < kStages; ++s)
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bars + 8 * s) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    const uint32_t chunks = len / 32, pairs = (uint32_t) (n / 64);
    const uint32_t first = blockIdx.x * (blockDim.x / 32) + warp;
    const uint32_t mine = first < pairs ? (pairs - first + warps - 1) / warps * chunks : 0;    // (pair, chunk) items
    for (uint32_t k = 0; k < kStages && k < mine; ++k)
        if (lane == 0)
            IssueTile(ring + k * kTileBytes, bars + 8 * k, &tm, (k % chunks) * 32, (first + k / chunks * warps) * 64);
    // 32B swizzle: the 16-byte half j of row r sits at r * 32 + 16 * (j ^ ((r >> 2) & 1))
    const uint32_t row = lane * 32, swz = (lane >> 2) & 1;
    uint32_t acc = 0;
    for (uint32_t k = 0; k < mine; ++k) {
        const uint32_t slot = k % kStages;
        MbarWait(bars + 8 * slot, (k / kStages) & 1);
        const uint32_t at = ring + slot * kTileBytes + row;
        uint4 v[4];
        for (int h = 0; h < 4; ++h)
            asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];"
                         : "=r"(v[h].x), "=r"(v[h].y), "=r"(v[h].z), "=r"(v[h].w)
                         : "r"(at + (h >> 1) * 1024 + 16 * ((h & 1) ^ swz))
                         : "memory");
        acc ^= Fold(v[0]) ^ Fold(v[1]) ^ Fold(v[2]) ^ Fold(v[3]);
        __syncwarp();
        const uint32_t next = k + kStages;
        if (lane == 0 && next < mine) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            IssueTile(ring + slot * kTileBytes, bars + 8 * slot, &tm, (next % chunks) * 32, (first + next / chunks * warps) * 64);
        }
    }
    if (acc == 0x12345678u)
        out[0] = acc;
}

// ---- per-lane cp.async ring: the input side of a two-string kernel that keeps kSlots 32-byte blocks of each string in
// shared memory (LDGSTS), read back with LDS.128.  One CTA per SM beside 76 KB held back for the hot table.  A slot of a
// warp is two 512-byte rows, one per 16-byte half, so that the copies and the reads of a warp are free of bank conflicts.
constexpr uint32_t kRingTableBytes = 76 * 1024;

// One 32-byte block into a slot: kCg = cp.async.cg (both halves to L2, L1 bypassed) or .ca (allocating in L1, so the
// second half is an L1 hit); the first half carries the kL2-byte prefetch-size hint.
template <bool kCg, int kL2>
__device__ __forceinline__ void CopyBlock(uint32_t dst, const uint8_t* src)
{
#define RING_COPY(LEVEL, HINT)                                                                                       \
    asm volatile("cp.async." LEVEL ".shared.global" HINT " [%0], [%1], 16;\n\t"                                     \
                 "cp.async." LEVEL ".shared.global [%2], [%3], 16;" ::"r"(dst), "l"(src), "r"(dst + 512), "l"(src + 16) \
                 : "memory")
    if (kCg && kL2 == 64)
        RING_COPY("cg", ".L2::64B");
    else if (kCg && kL2 == 128)
        RING_COPY("cg", ".L2::128B");
    else if (kCg)
        RING_COPY("cg", ".L2::256B");
    else if (kL2 == 64)
        RING_COPY("ca", ".L2::64B");
    else if (kL2 == 128)
        RING_COPY("ca", ".L2::128B");
    else
        RING_COPY("ca", ".L2::256B");
#undef RING_COPY
}

__device__ __forceinline__ uint4 Lds16(uint32_t at)
{
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(at) : "memory");
    return v;
}

template <bool kCg, int kL2, int kSlots>
__global__ void __launch_bounds__(1024, 1) LoadRingKernel(const uint8_t* corpus, uint64_t n, uint32_t len, uint32_t* out)
{
    extern __shared__ __align__(1024) uint8_t ring_smem[];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t) gridDim.x * (blockDim.x / 32);
    // slot k of string s (0, 1) of this lane: ring + (k * 2 + s) * 1024, second half 512 bytes further
    const uint32_t ring = (uint32_t) __cvta_generic_to_shared(ring_smem) + kRingTableBytes + warp * kSlots * 2048 + lane * 16;
    const uint32_t blocks = len / 32;
    uint32_t acc = 0;
    for (uint64_t pair = (uint64_t) blockIdx.x * (blockDim.x / 32) + warp; pair < n / 64; pair += warps) {
        const uint8_t* pa = corpus + (pair * 64 + lane) * (uint64_t) len;
        const uint8_t* pb = pa + 32 * (uint64_t) len;
#pragma unroll
        for (uint32_t k = 0; k < kSlots; ++k) {
            if (k < blocks) {
                CopyBlock<kCg, kL2>(ring + k * 2048, pa + 32 * k);
                CopyBlock<kCg, kL2>(ring + k * 2048 + 1024, pb + 32 * k);
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
        }
        uint32_t slot = 0;
        for (uint32_t k = 0; k < blocks; ++k) {
            asm volatile("cp.async.wait_group %0;" ::"n"(kSlots - 1) : "memory");
            const uint32_t at = ring + slot * 2048;
            const uint4 a0 = Lds16(at), a1 = Lds16(at + 512), b0 = Lds16(at + 1024), b1 = Lds16(at + 1536);
            if (k + kSlots < blocks) {
                CopyBlock<kCg, kL2>(at, pa + 32 * (k + kSlots));
                CopyBlock<kCg, kL2>(at + 1024, pb + 32 * (k + kSlots));
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
            acc ^= Fold(a0) ^ Fold(a1) ^ Fold(b0) ^ Fold(b1);
            slot = slot + 1 == kSlots ? 0 : slot + 1;
        }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    if (acc == 0x12345678u)
        out[0] = acc;
}

// The same ring with one string per lane (row 32u + lane of unit u): a warp's slot is 1 KB, two 512-byte rows (first and
// second 16-byte halves of 32 lanes), so the same shared memory buys twice the depth per string.
template <bool kCg, int kL2, int kSlots>
__global__ void __launch_bounds__(1024, 1) LoadRing1Kernel(const uint8_t* corpus, uint64_t n, uint32_t len, uint32_t* out)
{
    extern __shared__ __align__(1024) uint8_t ring_smem[];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t) gridDim.x * (blockDim.x / 32);
    const uint32_t ring = (uint32_t) __cvta_generic_to_shared(ring_smem) + kRingTableBytes + warp * kSlots * 1024 + lane * 16;
    const uint32_t blocks = len / 32;
    uint32_t acc = 0;
    for (uint64_t unit = (uint64_t) blockIdx.x * (blockDim.x / 32) + warp; unit < n / 32; unit += warps) {
        const uint8_t* p = corpus + (unit * 32 + lane) * (uint64_t) len;
#pragma unroll
        for (uint32_t k = 0; k < kSlots; ++k) {
            if (k < blocks)
                CopyBlock<kCg, kL2>(ring + k * 1024, p + 32 * k);
            asm volatile("cp.async.commit_group;" ::: "memory");
        }
        uint32_t slot = 0;
        for (uint32_t k = 0; k < blocks; ++k) {
            asm volatile("cp.async.wait_group %0;" ::"n"(kSlots - 1) : "memory");
            const uint32_t at = ring + slot * 1024;
            const uint4 a0 = Lds16(at), a1 = Lds16(at + 512);
            if (k + kSlots < blocks)
                CopyBlock<kCg, kL2>(at, p + 32 * (k + kSlots));
            asm volatile("cp.async.commit_group;" ::: "memory");
            acc ^= Fold(a0) ^ Fold(a1);
            slot = slot + 1 == kSlots ? 0 : slot + 1;
        }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    if (acc == 0x12345678u)
        out[0] = acc;
}

// mode 0: LDG.128 no_allocate, depth 1   mode 1: LDG.128 allocate (second half of the sector hits L1)
// mode 2: 2 x LDG.128 per 32 B, no_allocate   mode 3: 2 x LDG.128 per 32 B, allocating in L1
// mode 4: mode 3 with two 32-byte blocks in flight   mode 5: coalesced contiguous LDG.128 (upper bound)
template <int kMode>
__global__ void __launch_bounds__(512) LoadKernel(const uint8_t* corpus, uint64_t n, uint32_t len, uint32_t* out)
{
    const uint64_t warps = (uint64_t) gridDim.x * (blockDim.x / 32);
    const uint32_t lane = threadIdx.x & 31;
    uint32_t acc = 0;
    if (kMode == 5) {
        const uint64_t total16 = n * len / 16;
        for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < total16; i += (uint64_t) gridDim.x * blockDim.x)
            acc ^= Fold(Ld16(corpus + i * 16));
    } else {
        for (uint64_t unit = (uint64_t) blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); unit < n / 32; unit += warps) {
            const uint8_t* p = corpus + (unit * 32 + lane) * (uint64_t) len;
            if (kMode == 0 || kMode == 1) {
                uint4 cur = kMode == 0 ? Ld16(p) : Ld16Alloc(p);
                for (uint32_t off = 16; off < len; off += 16) {
                    uint4 nxt = kMode == 0 ? Ld16(p + off) : Ld16Alloc(p + off);
                    acc ^= Fold(cur);
                    cur = nxt;
                }
                acc ^= Fold(cur);
            } else if (kMode == 2 || kMode == 3) {
                uint4 a0, a1, b0, b1;
                Ld32<kMode == 3>(p, a0, a1);
                for (uint32_t off = 32; off < len; off += 32) {
                    Ld32<kMode == 3>(p + off, b0, b1);
                    acc ^= Fold(a0) ^ Fold(a1);
                    a0 = b0;
                    a1 = b1;
                }
                acc ^= Fold(a0) ^ Fold(a1);
            } else {
                uint4 a0, a1, b0, b1, c0, c1;
                Ld32<true>(p, a0, a1);
                Ld32<true>(p + 32, b0, b1);
                for (uint32_t off = 64; off < len; off += 32) {
                    Ld32<true>(p + off, c0, c1);
                    acc ^= Fold(a0) ^ Fold(a1);
                    a0 = b0; a1 = b1; b0 = c0; b1 = c1;
                }
                acc ^= Fold(a0) ^ Fold(a1) ^ Fold(b0) ^ Fold(b1);
            }
        }
    }
    if (acc == 0x12345678u)
        out[0] = acc;
}

// Do warp shuffles share the shared-memory data pipe?  kWhat: 1 = LDS.U8 chain only,
// 2 = SHFL chain only, 3 = both interleaved (two independent chains per thread).
// If the pipes were separate, mode 3 would take max(mode 1, mode 2); if shared, the sum.
template <int kWhat>
__global__ void __launch_bounds__(512) PipeKernel(uint32_t iters, uint32_t* out)
{
    __shared__ uint8_t table[8192];
    for (uint32_t i = threadIdx.x; i < 8192; i += blockDim.x)
        table[i] = (uint8_t) (i * 7 + 3);
    __syncthreads();
    uint32_t a = threadIdx.x & 255, b = threadIdx.x * 5 + 1, v = threadIdx.x;
    for (uint32_t i = 0; i < iters; ++i) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            if (kWhat & 1)
                a = table[(a << 5) | (threadIdx.x & 31)];          // conflict-free: bank = lane
            if (kWhat & 2)
                v = __shfl_sync(0xffffffffu, v + b, (v ^ k) & 31);
        }
    }
    if ((a ^ v) == 0xdeadbeefu)
        out[0] = a;
}

template <int kWhat>
void RunPipe(const char* name, uint32_t* out)
{
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    const uint32_t iters = 20000;
    PipeKernel<kWhat><<<sms * 3, 512>>>(iters, out);
    CK(cudaDeviceSynchronize());
    CK(cudaEventRecord(e0));
    PipeKernel<kWhat><<<sms * 3, 512>>>(iters, out);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    // warp-level ops of each kind per clock per SM, at the device's maximum SM clock
    int khz = 0;
    CK(cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0));
    double ops = (double) iters * 8 * 48;        // per SM: 48 warps
    std::printf("{\"bench\": \"pipe\", \"mode\": \"%s\", \"ms\": %.3f, \"warp_ops_per_clk_per_sm_each\": %.3f}\n", name, ms,
                ops / (ms * 1e-3 * khz * 1e3));
    std::fflush(stdout);
}

template <int kMode>
void Run(const char* name, const uint8_t* d, uint64_t n, uint32_t len, uint32_t* out, int threads_per_sm)
{
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    const int block = 512;
    const int grid = sms * (threads_per_sm / block);
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    for (int i = 0; i < 2; ++i)
        LoadKernel<kMode><<<grid, block>>>(d, n, len, out);
    CK(cudaDeviceSynchronize());
    float best = 1e30f;
    for (int rep = 0; rep < 5; ++rep) {
        CK(cudaEventRecord(e0));
        LoadKernel<kMode><<<grid, block>>>(d, n, len, out);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        best = ms < best ? ms : best;
    }
    std::printf("{\"bench\": \"load\", \"mode\": \"%s\", \"threads_per_sm\": %d, \"GBps\": %.1f, \"ms\": %.3f}\n", name,
                threads_per_sm, (double) n * len / best / 1e6, best);
    std::fflush(stdout);
}

void Report(const char* name, int threads_per_sm, uint64_t n, uint32_t len, float best)
{
    std::printf("{\"bench\": \"load\", \"mode\": \"%s\", \"threads_per_sm\": %d, \"GBps\": %.1f, \"ms\": %.3f}\n", name,
                threads_per_sm, (double) n * len / best / 1e6, best);
    std::fflush(stdout);
}

template <typename Launch>
float Best(Launch launch)
{
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    for (int i = 0; i < 2; ++i)
        launch();
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    float best = 1e30f;
    for (int rep = 0; rep < 5; ++rep) {
        CK(cudaEventRecord(e0));
        launch();
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        best = ms < best ? ms : best;
    }
    return best;
}

template <int kStages>
void RunTma(const char* name, const uint8_t* d, uint64_t n, uint32_t len, uint32_t* out)
{
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    using Encode = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    CK(cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &fn, 12000, cudaEnableDefault, &q));
    if (!fn || q != cudaDriverEntryPointSuccess) {
        std::fprintf(stderr, "cuTensorMapEncodeTiled unavailable\n");
        std::exit(1);
    }
    alignas(64) CUtensorMap tm;
    const cuuint64_t dims[2] = {len, n}, strides[1] = {len};
    const cuuint32_t box[2] = {32, 64}, estr[2] = {1, 1};
    CUresult r = reinterpret_cast<Encode>(fn)(&tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t*>(d), dims, strides, box, estr,
                                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        std::fprintf(stderr, "cuTensorMapEncodeTiled: %d\n", (int) r);
        std::exit(1);
    }
    const size_t smem = (size_t) 32 * kStages * kTileBytes + 32 * kStages * 8;
    CK(cudaFuncSetAttribute(TmaTileKernel<kStages>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
    Report(name, 1024, n, len, Best([&] { TmaTileKernel<kStages><<<sms, 1024, smem>>>(tm, n, len, out); }));
}

template <bool kCg, int kL2, int kSlots>
void RunRing(const uint8_t* d, uint64_t n, uint32_t len, uint32_t* out, int warps)
{
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    const size_t smem = kRingTableBytes + (size_t) warps * kSlots * 2048;
    CK(cudaFuncSetAttribute(LoadRingKernel<kCg, kL2, kSlots>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
    char name[96];
    std::snprintf(name, sizeof name, "ring_cp_async_%s_l2_%dB_%dwarps_%dslots", kCg ? "cg" : "ca", kL2, warps, kSlots);
    Report(name, warps * 32, n, len, Best([&] { LoadRingKernel<kCg, kL2, kSlots><<<sms, warps * 32, smem>>>(d, n, len, out); }));
}

template <bool kCg, int kL2>
void RunRingShapes(const uint8_t* d, uint64_t n, uint32_t len, uint32_t* out)
{
    RunRing<kCg, kL2, 2>(d, n, len, out, 32);
    RunRing<kCg, kL2, 2>(d, n, len, out, 28);
    RunRing<kCg, kL2, 3>(d, n, len, out, 24);
}

template <bool kCg, int kL2, int kSlots>
void RunRing1(const uint8_t* d, uint64_t n, uint32_t len, uint32_t* out, int warps)
{
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    const size_t smem = kRingTableBytes + (size_t) warps * kSlots * 1024;
    CK(cudaFuncSetAttribute(LoadRing1Kernel<kCg, kL2, kSlots>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
    char name[96];
    std::snprintf(name, sizeof name, "ring1_cp_async_%s_l2_%dB_%dwarps_%dslots", kCg ? "cg" : "ca", kL2, warps, kSlots);
    Report(name, warps * 32, n, len, Best([&] { LoadRing1Kernel<kCg, kL2, kSlots><<<sms, warps * 32, smem>>>(d, n, len, out); }));
}

// One string per lane at (warps, slots) = (16, 8), (24, 4), (24, 6), (32, 3), (32, 4): 96 to 144 KB of ring.
template <int kL2>
void RunRing1Shapes(const uint8_t* d, uint64_t n, uint32_t len, uint32_t* out)
{
    RunRing1<true, kL2, 8>(d, n, len, out, 16);
    RunRing1<true, kL2, 4>(d, n, len, out, 24);
    RunRing1<true, kL2, 6>(d, n, len, out, 24);
    RunRing1<true, kL2, 3>(d, n, len, out, 32);
    RunRing1<true, kL2, 4>(d, n, len, out, 32);
}

// The shipped two-string ring next to the one-string shapes, and the two-string ring at 16 x 4 (the same 128 KB spent on
// fewer strings), alternated twice so that drift between rows shows.
void RunRingComparison(const uint8_t* d, uint64_t n, uint32_t len, uint32_t* out)
{
    for (int pass = 0; pass < 2; ++pass) {
        RunRing<true, 128, 3>(d, n, len, out, 24);
        RunRing<true, 128, 4>(d, n, len, out, 16);
        RunRing1Shapes<128>(d, n, len, out);
        RunRing1Shapes<256>(d, n, len, out);
    }
}

int main(int argc, char** argv)
{
    const double gib = argc > 1 ? std::atof(argv[1]) : 4.0;
    const uint32_t len = argc > 2 ? (uint32_t) std::atoi(argv[2]) : 1024;
    const uint64_t n = (uint64_t) (gib * (1ull << 30) / len) / 64 * 64;
    uint8_t* d;
    uint32_t* out;
    CK(cudaMalloc(&d, n * len));
    CK(cudaMalloc(&out, 64));
    CK(cudaMemset(d, 0x5a, n * len));
    if (argc > 3 && std::strcmp(argv[3], "ring") == 0) {
        RunRingComparison(d, n, len, out);
        return 0;
    }
    RunPipe<1>("lds_only", out);
    RunPipe<2>("shfl_only", out);
    RunPipe<3>("lds_and_shfl", out);
    if (argc > 3)
        return 0;
    {
        int sms = 0;
        CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
        // the flagship's shapes first, each next to the coalesced bound at the same residency
        Run<5>("coalesced_ldg128", d, n, len, out, 1024);
        Report("flagship_lane_2xldg128_l1_two_strings", 896, n, len, Best([&] { LoadPairKernel<0><<<sms * 2, 448>>>(d, n, len, out); }));
        Report("two_strings_l2_64B", 896, n, len, Best([&] { LoadPairKernel<64><<<sms * 2, 448>>>(d, n, len, out); }));
        Report("two_strings_l2_128B", 896, n, len, Best([&] { LoadPairKernel<128><<<sms * 2, 448>>>(d, n, len, out); }));
        Report("two_strings_l2_256B", 896, n, len, Best([&] { LoadPairKernel<256><<<sms * 2, 448>>>(d, n, len, out); }));
        RunTma<2>("flagship_tma_tile_64x32_swz32_2stages", d, n, len, out);
        RunTma<3>("tma_tile_64x32_swz32_3stages", d, n, len, out);
        // two strings per lane fed from a per-lane cp.async ring, at (warps, slots) = (32, 2), (28, 2), (24, 3)
        RunRingShapes<false, 64>(d, n, len, out);
        RunRingShapes<false, 128>(d, n, len, out);
        RunRingShapes<false, 256>(d, n, len, out);
        RunRingShapes<true, 64>(d, n, len, out);
        RunRingShapes<true, 128>(d, n, len, out);
        RunRingShapes<true, 256>(d, n, len, out);
    }
    for (int tps : {1024, 1536, 2048}) {
        Run<5>("coalesced_ldg128", d, n, len, out, tps);
        Run<0>("lane_ldg128_noalloc", d, n, len, out, tps);
        Run<1>("lane_ldg128_l1", d, n, len, out, tps);
        Run<2>("lane_2xldg128_noalloc", d, n, len, out, tps);
        Run<3>("lane_2xldg128_l1", d, n, len, out, tps);
        Run<4>("lane_2xldg128_l1_depth2", d, n, len, out, tps);
    }
    return 0;
}
