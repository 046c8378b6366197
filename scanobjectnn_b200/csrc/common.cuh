// common.cuh -- shared helpers for libpsa.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/psa.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ < 900)
#error "libpsa is written for sm_90a (H100) only"
#endif

namespace psa {

constexpr int kNumSMs = 132;  // H100 SXM

void set_error(const char* fmt, ...);

// scatter.cu: stable counting sort of a cloud's (entry -> destination) pairs; offsets (b, n+1), list (b, mk)
int launch_group_csr(int b, int n, int mk, const int* idx, int* offsets, int* list, cudaStream_t st);

// train.cu: out[e] = sum_p partial[p * len + e] in a fixed order (fp64)
int reduce_partials(int nparts, int len, const float* partial, float* out, cudaStream_t st);
// train.cu: the contraction split of a weight gradient over `rows` rows with `tiles` output tiles (splits, rows per split)
int weight_grad_splits(long long rows, int tiles, long long* k_per_split);
// train.cu: batch-norm backward from (nparts, 2, C) partials [sum dz | sum dz * xhat] over `rows` rows -> dgamma, dbeta and the
// coefficients of dy = ca * dz + cb * y + cc (psa_bn_bwd_coeffs)
int launch_bn_bwd_final(int nparts, int C, long long rows, const float* partial, const float* gamma, const float* mean_inv, float* dgamma,
                        float* dbeta, float* ca, float* cb, float* cc, cudaStream_t st);

inline int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return (int)e;
    }
    return PSA_OK;
}

#define PSA_REQUIRE(cond, ...)                \
    do {                                      \
        if (!(cond)) {                        \
            ::psa::set_error(__VA_ARGS__);    \
            return PSA_ERR_INVALID_ARGUMENT;  \
        }                                     \
    } while (0)

#define PSA_SUPPORTED(cond, ...)              \
    do {                                      \
        if (!(cond)) {                        \
            ::psa::set_error(__VA_ARGS__);    \
            return PSA_ERR_UNSUPPORTED;       \
        }                                     \
    } while (0)

#define PSA_CUDA(call)                                                      \
    do {                                                                    \
        cudaError_t e_ = (call);                                            \
        if (e_ != cudaSuccess) {                                            \
            ::psa::set_error("%s: %s", #call, cudaGetErrorString(e_));      \
            return (int)e_;                                                 \
        }                                                                   \
    } while (0)

static inline cudaStream_t as_stream(psa_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

// Squared distance exactly as the reference's CUDA kernels evaluate it after nvcc's FMA contraction
// (SASS of tf_sampling_g.cu / tf_grouping_g.cu: FMUL dy*dy ; FFMA dx,dx ; FFMA dz,dz).
__device__ __forceinline__ float dist2_ref_gpu(float dx, float dy, float dz) {
    float t = __fmul_rn(dy, dy);
    t = __fmaf_rn(dx, dx, t);
    t = __fmaf_rn(dz, dz, t);
    return t;
}
// Squared distance exactly as the reference's CPU ops (x86-64, no FMA) evaluate it: (dx*dx+dy*dy)+dz*dz.
__device__ __forceinline__ float dist2_ref_cpu(float dx, float dy, float dz) {
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// Cooperative copy of `count` floats global -> shared with 8 independent loads in flight per thread (a plain
// `for (i) s[i] = g[i]` loop is one L2 round trip per iteration: ~0.35 us each, tens of us for a 24 KB cloud).
template <int THREADS>
__device__ __forceinline__ void stage_floats(float* __restrict__ dst, const float* __restrict__ src, int count, int tid) {
    int i = tid;
    for (; i + 7 * THREADS < count; i += 8 * THREADS) {
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = __ldg(src + i + u * THREADS);
#pragma unroll
        for (int u = 0; u < 8; ++u) dst[i + u * THREADS] = v[u];
    }
    for (; i < count; i += THREADS) dst[i] = __ldg(src + i);
}

// Two-lane float arithmetic, each lane rounded on its own (identical results to two scalar __f*_rn calls).
__device__ __forceinline__ float2 fadd2_rn(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2_rn(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 ffma2_rn(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }

__device__ __forceinline__ unsigned lanemask_lt() {
    unsigned m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

}  // namespace psa
