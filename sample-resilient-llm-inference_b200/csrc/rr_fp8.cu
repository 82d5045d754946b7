// rr_fp8.cu — FP8 weights: the per-row quantizer and the dequantizer of the e4m3 projection weights.
//
// A weight W [N, K] bf16 is stored as Q [N, K] e4m3 (row-major, row pitch K bytes) and one fp32 scale per row,
// s[n] = 2^e[n], with
//   e[n] = the smallest integer with max_k |W[n, k]| <= 448 * 2^e, clamped to [-117, 127] (0 for an all-zero row),
//   Q    = e4m3_rne(W / 2^e[n])   (subnormals included; |W / 2^e| <= 448, so it never saturates).
// D = bf16(Q * s) is exact (e4m3_to_bf16x4 in rr_ptx.cuh): every e4m3 value times a power of two in that range is a
// normal bf16, except for the largest codes of a row whose amax lies within 2^-4 of bf16's largest value, which the
// quantizer refuses.  The decode GEMMs convert Q tiles into D tiles in shared memory (rr_gemm.cu); prefill runs its bf16 GEMMs
// on D, written here into an engine-owned scratch once per layer and chunk.  Both kernels are bandwidth-bound copies.
#include "rr_kernels.h"
#include "rr_launch.cuh"
#include "rr_ptx.cuh"

#include <cuda_fp8.h>

namespace rr {
namespace {

constexpr int QZ_WARPS = 8;

// One warp per row: amax and finiteness over the row, then the scaled conversion (the second pass reads from L1 / L2).  A row
// with Inf or NaN, or whose largest value rounds to an e4m3 code that times 2^e leaves the bf16 range (amax within 2^-4 of
// bf16's largest value), sets *bad and writes nothing: D = bf16(Q * s) would not be exact.
__global__ void __launch_bounds__(QZ_WARPS * 32)
quantize_fp8_kernel(const __nv_bfloat16* __restrict__ w, int rows, int K, int ld, uint8_t* __restrict__ q,
                    float* __restrict__ scale, int* __restrict__ bad) {
    griddep_launch();
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * QZ_WARPS + (threadIdx.x >> 5);
    if (row >= rows) return;
    const __nv_bfloat16* src = w + (size_t)row * ld;
    griddep_wait();
    float a = 0.f;
    bool finite = true;
    for (int k = 8 * lane; k < K; k += 256) {
        const uint4 v = *reinterpret_cast<const uint4*>(src + k);
        const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float f0 = bf16_lo(u[j]), f1 = bf16_hi(u[j]);
            finite = finite && isfinite(f0) && isfinite(f1);
            a = fmaxf(a, fmaxf(fabsf(f0), fabsf(f1)));
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, o));
    if (!__all_sync(0xffffffffu, finite)) {
        if (lane == 0) atomicExch(bad, 1);
        return;
    }
    int e = 0;
    if (a > 0.f) {
        int E;
        frexpf(a, &E);                                   // a in [2^(E-1), 2^E): 448 * 2^(E-10) < a <= 448 * 2^(E-8)
        e = E - 9;
        if (a > ldexpf(448.f, e)) ++e;
        e = e < -117 ? -117 : (e > 127 ? 127 : e);
    }
    const float inv = ldexpf(1.f, -e);                  // exact: W / 2^e
    const float qmax = __half2float(__nv_cvt_fp8_to_halfraw(__nv_cvt_float_to_fp8(a * inv, __NV_SATFINITE, __NV_E4M3),
                                                            __NV_E4M3));
    if (qmax * ldexpf(1.f, e) > 3.3895313892515355e38f) {   // bf16's largest finite value; beyond it the product is inf
        if (lane == 0) atomicExch(bad, 1);
        return;
    }
    uint8_t* dst = q + (size_t)row * K;
    for (int k = 8 * lane; k < K; k += 256) {
        const uint4 v = *reinterpret_cast<const uint4*>(src + k);
        const uint32_t u[4] = {v.x, v.y, v.z, v.w};
        uint32_t out[2];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const __nv_fp8x2_storage_t lo = __nv_cvt_float2_to_fp8x2(
                make_float2(bf16_lo(u[2 * j]) * inv, bf16_hi(u[2 * j]) * inv), __NV_SATFINITE, __NV_E4M3);
            const __nv_fp8x2_storage_t hi = __nv_cvt_float2_to_fp8x2(
                make_float2(bf16_lo(u[2 * j + 1]) * inv, bf16_hi(u[2 * j + 1]) * inv), __NV_SATFINITE, __NV_E4M3);
            out[j] = (uint32_t)lo | ((uint32_t)hi << 16);
        }
        *reinterpret_cast<uint2*>(dst + k) = make_uint2(out[0], out[1]);
    }
    if (lane == 0) scale[row] = ldexpf(1.f, e);
}

// 16 e4m3 values of one row per thread and step -> 32 bytes of bf16(Q * s); grid-stride over the chunks of every job.
__global__ void __launch_bounds__(256)
dequantize_fp8_kernel(const __grid_constant__ Fp8DequantJobs J) {
    const long long total = J.end[J.n - 1];
    for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < total; c += (long long)gridDim.x * blockDim.x) {
        int i = 0;
        while (c >= J.end[i]) ++i;
        const Fp8DequantJob& j = J.job[i];
        const long long lc = c - (i ? J.end[i - 1] : 0);
        const int per_row = j.K / 16;
        const int row = (int)(lc / per_row), col = (int)(lc - (long long)row * per_row) * 16;
        const uint4 v = *reinterpret_cast<const uint4*>(j.q + (size_t)row * j.K + col);
        const float s = j.scale[row];
        const uint2 a = e4m3x4_to_bf16x4(v.x, s), b = e4m3x4_to_bf16x4(v.y, s);
        const uint2 c2 = e4m3x4_to_bf16x4(v.z, s), d = e4m3x4_to_bf16x4(v.w, s);
        uint4* dst = reinterpret_cast<uint4*>(j.out + (size_t)row * j.ld_out + col);
        dst[0] = make_uint4(a.x, a.y, b.x, b.y);
        dst[1] = make_uint4(c2.x, c2.y, d.x, d.y);
    }
}

}  // namespace

bool fp8_weight_ok(const void* q, int K) { return q && ((uintptr_t)q & 15) == 0 && K >= 16 && K % 16 == 0; }

int launch_quantize_fp8(const __nv_bfloat16* w, int rows, int K, int ld, uint8_t* q, float* scale, int* bad, cudaStream_t st) {
    const int grid = (rows + QZ_WARPS - 1) / QZ_WARPS;
    const cudaError_t e = launch_pdl(quantize_fp8_kernel, dim3(grid), dim3(QZ_WARPS * 32), 0, st, w, rows, K, ld, q, scale, bad);
    return e == cudaSuccess ? RR_OK : RR_ERR_CUDA;
}

// A plain (stream-ordered) launch: it starts after every earlier kernel of the stream has finished, and the kernel does not
// trigger its dependents, so nothing after it starts before its last write (DESIGN §4, the prefill scratch).
int launch_dequantize_fp8(const Fp8DequantJobs& J, cudaStream_t st) {
    if (J.n < 1 || J.n > 4 || J.end[J.n - 1] <= 0) return RR_ERR_ARG;
    long long grid = (J.end[J.n - 1] + 255) / 256;
    if (grid > 8LL * num_sms()) grid = 8LL * num_sms();
    dequantize_fp8_kernel<<<(int)grid, 256, 0, st>>>(J);
    return cudaGetLastError() == cudaSuccess ? RR_OK : RR_ERR_CUDA;
}

void fp8_dequant_job(Fp8DequantJobs* J, const void* q, const float* scale, int rows, int K, __nv_bfloat16* out, int ld_out) {
    Fp8DequantJob& j = J->job[J->n];
    j.q = (const uint8_t*)q; j.scale = scale; j.out = out; j.rows = rows; j.K = K; j.ld_out = ld_out;
    J->end[J->n] = (J->n ? J->end[J->n - 1] : 0) + (long long)rows * (K / 16);
    ++J->n;
}

}  // namespace rr
