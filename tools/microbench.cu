// tools/microbench.cu -- how fast can one-string-per-lane loads pull a corpus of
// 1 KiB strings out of HBM?  Measures the load path of the scan kernel in
// isolation (XOR-reduce, no table walk) for several load shapes, so that the
// scan kernel's distance from the HBM roofline can be attributed to the walk
// (shared-memory wavefronts) or to the loads (L1TEX tag stage: 32 distinct
// lines per warp-wide request).  Not part of the product library.
//
//   microbench [GiB=4] [string_len=1024]
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
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

int main(int argc, char** argv)
{
    const double gib = argc > 1 ? std::atof(argv[1]) : 4.0;
    const uint32_t len = argc > 2 ? (uint32_t) std::atoi(argv[2]) : 1024;
    const uint64_t n = (uint64_t) (gib * (1ull << 30) / len) / 32 * 32;
    uint8_t* d;
    uint32_t* out;
    CK(cudaMalloc(&d, n * len));
    CK(cudaMalloc(&out, 64));
    CK(cudaMemset(d, 0x5a, n * len));
    RunPipe<1>("lds_only", out);
    RunPipe<2>("shfl_only", out);
    RunPipe<3>("lds_and_shfl", out);
    if (argc > 3)
        return 0;
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
