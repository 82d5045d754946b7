// hbm_read_probe.cu — how fast can the SMs READ HBM, and does the tile shape matter?
//   (a) plain 16-byte loads, grid-stride                                  (upper bound of a read-only stream)
//   (b) TMA 2-D boxes of 128 rows x 128 B out of a [N, K] bf16 matrix     (what the decode GEMMs request today)
//   (c) TMA 2-D boxes of the same 16 KB out of a pre-tiled [N*K/64, 64] matrix = one contiguous 16 KB block
// (b)/(c): one elected thread per CTA keeps DEPTH boxes in flight and recycles a slot as soon as it lands.
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o build/hbm_read_probe tools/probes/hbm_read_probe.cu
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e)); exit(1); } } while (0)

__global__ void read_ld(const uint4* __restrict__ p, size_t n, unsigned* sink) {
    uint4 acc = make_uint4(0, 0, 0, 0);
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t step = (size_t)gridDim.x * blockDim.x;
    for (; i + 3 * step < n; i += 4 * step) {
        uint4 a = __ldcs(p + i), b = __ldcs(p + i + step), c = __ldcs(p + i + 2 * step), d = __ldcs(p + i + 3 * step);
        acc.x ^= a.x ^ b.x ^ c.x ^ d.x; acc.y ^= a.y ^ b.y ^ c.y ^ d.y; acc.z ^= a.z ^ b.z ^ c.z ^ d.z; acc.w ^= a.w ^ b.w ^ c.w ^ d.w;
    }
    for (; i < n; i += step) { uint4 a = __ldcs(p + i); acc.x ^= a.x; acc.y ^= a.y; acc.z ^= a.z; acc.w ^= a.w; }
    if ((acc.x ^ acc.y ^ acc.z ^ acc.w) == 0x12345678u) *sink = 1;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

template <int DEPTH>
__global__ void __launch_bounds__(32, 1) read_tma(const __grid_constant__ CUtensorMap tm, int tiles, int kblocks, int tiled, int ahead) {
    extern __shared__ uint8_t raw[];
    uint8_t* sm = (uint8_t*)(((uintptr_t)raw + 1023) & ~(uintptr_t)1023);
    uint64_t* bar = (uint64_t*)(sm + DEPTH * 16384);
    if (threadIdx.x != 0) return;
    for (int s = 0; s < DEPTH; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(bar + s)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    int st = 0; uint32_t par = 0; long long issued = 0;
    for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
        for (int kb = 0; kb < kblocks; ++kb, ++issued) {
            if (issued >= DEPTH) {
                uint32_t ok = 0;
                while (!ok)
                    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                                 : "=r"(ok) : "r"(smem_u32(bar + st)), "r"(par) : "memory");
            }
            if (ahead > 0) {          // L2 prefetch of the box `ahead` positions further along this CTA's stream (same tile only)
                const int kp = kb + ahead;
                if (kp < kblocks) {
                    const int p0 = tiled ? 0 : kp * 64, p1 = tiled ? (t * kblocks + kp) * 128 : t * 128;
                    asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"((uint64_t)&tm), "r"(p0), "r"(p1) : "memory");
                }
            }
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar + st)), "r"(16384) : "memory");
            const int c0 = tiled ? 0 : kb * 64;
            const int c1 = tiled ? (t * kblocks + kb) * 128 : t * 128;
            asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
                         ::"r"(smem_u32(sm + st * 16384)), "l"((uint64_t)&tm), "r"(smem_u32(bar + st)), "r"(c0), "r"(c1), "l"(pol) : "memory");
            if (++st == DEPTH) { st = 0; par ^= (issued >= DEPTH) ? 1u : 0u; }
        }
    }
    // drain
    long long left = issued < DEPTH ? issued : DEPTH;
    for (long long i = 0; i < left; ++i) {
        uint32_t ok = 0;
        while (!ok)
            asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                         : "=r"(ok) : "r"(smem_u32(bar + st)), "r"(par) : "memory");
        if (++st == DEPTH) { st = 0; par ^= 1u; }
    }
}


// (d) the decode GEMM's request mix: every 16 KB weight box is accompanied by an activation box of XROWS x 128 B that is
// re-read by every CTA (L2 hits).  Does the L2 -> SM path carry both at the HBM rate?
template <int DEPTH, int XROWS>
__global__ void __launch_bounds__(32, 1) read_tma_wx(const __grid_constant__ CUtensorMap tm, const __grid_constant__ CUtensorMap tx,
                                                     int tiles, int kblocks) {
    extern __shared__ uint8_t raw[];
    constexpr int XB = XROWS * 128, ST = 16384 + (XB > 0 ? ((XB + 1023) / 1024 * 1024) : 0);
    uint8_t* sm = (uint8_t*)(((uintptr_t)raw + 1023) & ~(uintptr_t)1023);
    uint64_t* bar = (uint64_t*)(sm + DEPTH * ST);
    if (threadIdx.x != 0) return;
    for (int s = 0; s < DEPTH; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(bar + s)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    uint64_t pol, polx;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(polx));
    int st = 0; uint32_t par = 0; long long issued = 0;
    for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
        for (int kb = 0; kb < kblocks; ++kb, ++issued) {
            if (issued >= DEPTH) {
                uint32_t ok = 0;
                while (!ok)
                    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                                 : "=r"(ok) : "r"(smem_u32(bar + st)), "r"(par) : "memory");
            }
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar + st)), "r"(16384 + XB) : "memory");
            asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
                         ::"r"(smem_u32(sm + st * ST)), "l"((uint64_t)&tm), "r"(smem_u32(bar + st)), "r"(kb * 64), "r"(t * 128), "l"(pol) : "memory");
            if (XB > 0)
                asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
                             ::"r"(smem_u32(sm + st * ST + 16384)), "l"((uint64_t)&tx), "r"(smem_u32(bar + st)), "r"(kb * 64), "r"(0), "l"(polx) : "memory");
            if (++st == DEPTH) { st = 0; par ^= (issued >= DEPTH) ? 1u : 0u; }
        }
    }
    long long left = issued < DEPTH ? issued : DEPTH;
    for (long long i = 0; i < left; ++i) {
        uint32_t ok = 0;
        while (!ok)
            asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                         : "=r"(ok) : "r"(smem_u32(bar + st)), "r"(par) : "memory");
        if (++st == DEPTH) { st = 0; par ^= 1u; }
    }
}
template <int DEPTH, int XROWS>
static float run_wx(const CUtensorMap& tm, const CUtensorMap& tx, int tiles, int kblocks, int grid, int iters) {
    constexpr int XB = XROWS * 128, ST = 16384 + (XB > 0 ? ((XB + 1023) / 1024 * 1024) : 0);
    const int smem = DEPTH * ST + 1024 + 256;
    CK(cudaFuncSetAttribute(read_tma_wx<DEPTH, XROWS>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    read_tma_wx<DEPTH, XROWS><<<grid, 32, smem>>>(tm, tx, tiles, kblocks);
    CK(cudaDeviceSynchronize());
    cudaEventRecord(e0);
    for (int i = 0; i < iters; ++i) read_tma_wx<DEPTH, XROWS><<<grid, 32, smem>>>(tm, tx, tiles, kblocks);
    cudaEventRecord(e1);
    CK(cudaDeviceSynchronize());
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    return ms / iters;
}

typedef CUresult (*PFN_enc)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                            const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static CUtensorMap mk(PFN_enc enc, void* base, uint64_t rows, uint64_t K, int promo, int box_rows = 128) {
    CUtensorMap m;
    cuuint64_t dims[2] = {K, rows};
    cuuint64_t str[1] = {K * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, dims, str, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     promo ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { printf("encode failed %d\n", (int)r); exit(1); }
    return m;
}

template <int DEPTH>
static float run_tma(const CUtensorMap& tm, int tiles, int kblocks, int tiled, int grid, int iters, int ahead = 0) {
    const int smem = DEPTH * 16384 + 1024 + 256;
    CK(cudaFuncSetAttribute(read_tma<DEPTH>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    read_tma<DEPTH><<<grid, 32, smem>>>(tm, tiles, kblocks, tiled, ahead);
    CK(cudaDeviceSynchronize());
    cudaEventRecord(e0);
    for (int i = 0; i < iters; ++i) read_tma<DEPTH><<<grid, 32, smem>>>(tm, tiles, kblocks, tiled, ahead);
    cudaEventRecord(e1);
    CK(cudaDeviceSynchronize());
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    return ms / iters;
}

int main() {
    void* fp = nullptr; cudaDriverEntryPointQueryResult q;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q));
    PFN_enc enc = (PFN_enc)fp;
    int sms; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    const uint64_t N = 128 * 1024, K = 8192;            // 2 GiB of bf16: far beyond the 126 MB L2
    const size_t bytes = N * K * 2;
    void* buf; CK(cudaMalloc(&buf, bytes)); CK(cudaMemset(buf, 1, bytes));
    unsigned* sink; CK(cudaMalloc(&sink, 4));
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int bpsm : {8, 16, 32}) for (int thr : {256, 512}) {
        read_ld<<<sms * bpsm, thr>>>((const uint4*)buf, bytes / 16, sink);
        CK(cudaDeviceSynchronize());
        cudaEventRecord(e0);
        for (int i = 0; i < 5; ++i) read_ld<<<sms * bpsm, thr>>>((const uint4*)buf, bytes / 16, sink);
        cudaEventRecord(e1); CK(cudaDeviceSynchronize());
        float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= 5;
        printf("ld.128 grid-stride  %2d CTAs/SM x %3d thr : %7.1f us  %6.0f GB/s\n", bpsm, thr, ms * 1e3, bytes / ms / 1e6);
    }
    for (uint64_t Kv : {4096ull, 14336ull}) {
        const uint64_t rows = (bytes / 2 / Kv) / 128 * 128;
        const int tiles = (int)(rows / 128), kblocks = (int)(Kv / 64);
        const double b = (double)tiles * kblocks * 16384;
        for (int promo : {1, 0}) {
            CUtensorMap strided = mk(enc, buf, rows, Kv, promo);
            CUtensorMap tiled = mk(enc, buf, (uint64_t)tiles * kblocks * 128, 64, promo);
            float a8 = run_tma<8>(strided, tiles, kblocks, 0, sms, 5), a12 = run_tma<12>(strided, tiles, kblocks, 0, sms, 5);
            float t8 = run_tma<8>(tiled, tiles, kblocks, 1, sms, 5), t12 = run_tma<12>(tiled, tiles, kblocks, 1, sms, 5);
            printf("TMA K=%5llu promo256=%d: strided depth 8 %6.0f GB/s, depth 12 %6.0f | pre-tiled depth 8 %6.0f GB/s, depth 12 %6.0f\n",
                   (unsigned long long)Kv, promo, b / a8 / 1e6, b / a12 / 1e6, b / t8 / 1e6, b / t12 / 1e6);
        }
    }
    {   // shallow smem ring + L2 look-ahead: can 4 slots (64 KB in flight per SM) keep the stream at full rate?
        const uint64_t Kv = 4096, rows = (bytes / 2 / Kv) / 128 * 128;
        const int tiles = (int)(rows / 128), kblocks = (int)(Kv / 64);
        const double b = (double)tiles * kblocks * 16384;
        CUtensorMap strided = mk(enc, buf, rows, Kv, 1);
        for (int ahead : {0, 4, 8, 12, 16, 24}) {
            float d2 = run_tma<2>(strided, tiles, kblocks, 0, sms, 5, ahead), d3 = run_tma<3>(strided, tiles, kblocks, 0, sms, 5, ahead),
                  d4 = run_tma<4>(strided, tiles, kblocks, 0, sms, 5, ahead), d8 = run_tma<8>(strided, tiles, kblocks, 0, sms, 5, ahead);
            printf("TMA strided K=4096, L2 prefetch %2d boxes ahead: ring 2 %6.0f  ring 3 %6.0f  ring 4 %6.0f  ring 8 %6.0f GB/s\n", ahead,
                   b / d2 / 1e6, b / d3 / 1e6, b / d4 / 1e6, b / d8 / 1e6);
        }
    }
    {   // fewer CTAs than SMs (the second gate/up wave of the fused MLP runs on 76, the late down items on ~96): is a lone CTA's
        // rate set by its ring depth (bytes in flight / latency)?
        const uint64_t Kv = 4096, rows = (bytes / 2 / Kv) / 128 * 128;
        const int tiles = (int)(rows / 128) / 4, kblocks = (int)(Kv / 64);
        const double b = (double)tiles * kblocks * 16384;
        CUtensorMap strided = mk(enc, buf, rows, Kv, 1);
        for (int g : {32, 66, 96, 132}) {
            float d6 = run_tma<6>(strided, tiles, kblocks, 0, g, 3), d8 = run_tma<8>(strided, tiles, kblocks, 0, g, 3),
                  d10 = run_tma<10>(strided, tiles, kblocks, 0, g, 3), d12 = run_tma<12>(strided, tiles, kblocks, 0, g, 3);
            printf("%3d CTAs: ring 6 %5.1f  ring 8 %5.1f  ring 10 %5.1f  ring 12 %5.1f GB/s per SM\n", g, b / d6 / 1e6 / g, b / d8 / 1e6 / g,
                   b / d10 / 1e6 / g, b / d12 / 1e6 / g);
        }
    }
    {   // weight stream + re-read activation stream
        const uint64_t Kv = 4096, rows = (bytes / 2 / Kv) / 128 * 128;
        const int tiles = (int)(rows / 128), kblocks = (int)(Kv / 64);
        const double b = (double)tiles * kblocks * 16384;
        CUtensorMap w = mk(enc, buf, rows, Kv, 1);
        void* xb; CK(cudaMalloc(&xb, 64 * Kv * 2)); CK(cudaMemset(xb, 1, 64 * Kv * 2));
        CUtensorMap x64 = mk(enc, xb, 64, Kv, 1, 64), x32 = mk(enc, xb, 64, Kv, 1, 32), x16 = mk(enc, xb, 64, Kv, 1, 16);
        float t0 = run_wx<8, 0>(w, x64, tiles, kblocks, sms, 5), t64 = run_wx<8, 64>(w, x64, tiles, kblocks, sms, 5),
              t32 = run_wx<8, 32>(w, x32, tiles, kblocks, sms, 5), t16 = run_wx<8, 16>(w, x16, tiles, kblocks, sms, 5),
              t32d = run_wx<10, 32>(w, x32, tiles, kblocks, sms, 5);
        printf("W stream (16 KB boxes, ring 8) alone %6.0f GB/s | + 8 KB activation box %6.0f | + 4 KB %6.0f | + 2 KB %6.0f | + 4 KB, ring 10 %6.0f\n",
               b / t0 / 1e6, b / t64 / 1e6, b / t32 / 1e6, b / t16 / 1e6, b / t32d / 1e6);
    }
    return 0;
}
