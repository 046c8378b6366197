// sampling.cu -- farthest point sampling + gather_point (+grad) for sm_90a.
//
// Replaces pointnet2/tf_ops/sampling/tf_sampling_g.cu:105-192 of the reference.  Results are index-exact with the
// reference kernel, including its tie-break (minimum over (k mod 512, k) among equal maxima), which is carried as an
// explicit 32-bit key so the thread <-> point mapping is free.  One CTA per cloud with as FEW warps as the registers
// allow (4 warps up to N=2048: the round time is dominated by the cross-warp arg-max, not by arithmetic); coordinates
// and running min-distances live in registers (no global `temp` round trip), distances are computed on float pairs
// (same IEEE operations and order as the reference's contraction), the block arg-max is
// REDUX.MAX + REDUX.MIN per warp and one shared-memory hop (1 __syncthreads per round instead of the reference's 10),
// and the gather of the sampled coordinates is fused.
#include <limits.h>

#include "common.cuh"

namespace psa {

// The reference's tie-break: thread t of its 512-thread block scans k = t, t+512, ... with strict '>', then a tree that
// keeps the lower slot, i.e. the winner among equal maxima is the minimum over (k mod 512, k).  Encoded as one
// unsigned key so that any thread <-> point mapping can reproduce it with REDUX.MAX(value) + REDUX.MIN(key).
__device__ __forceinline__ unsigned fps_tie_key(int k) { return ((unsigned)(k & 511) << 22) | (unsigned)(k >> 9); }
__device__ __forceinline__ int fps_key_to_index(unsigned key) { return (int)((key >> 22) | ((key & 0x3fffffu) << 9)); }

// T threads per cloud, each owning S = 512/T reference slots with R points per slot (PPT = S*R, n <= 512*R).
// The thread's points are ordered by increasing tie key (slot-major), so a strict '>' scan keeps the right one on ties.
template <int T, int R>
__global__ void __launch_bounds__(T, 1)
fps_kernel(int n, int m, const float* __restrict__ xyz, int* __restrict__ idx_out, float* __restrict__ new_xyz) {
    constexpr int S = 512 / T, PPT = S * R, W = T / 32;
    constexpr int NP = (PPT + 1) / 2;                              // points are processed in packed pairs
    extern __shared__ float smem_f[];
    float* sxyz = smem_f;                                          // n*3 floats, flat copy of the cloud
    int* s_sel = reinterpret_cast<int*>(smem_f + (size_t)n * 3);   // m selected indices
    __shared__ int s_wval[2][W];
    __shared__ unsigned s_wkey[2][W];

    const int cloud = blockIdx.x;
    const int t = threadIdx.x;
    const int lane = t & 31, warp = t >> 5;
    const float* p = xyz + (size_t)cloud * n * 3;
    stage_floats<T>(sxyz, p, n * 3, t);
    __syncthreads();

    float2 px[NP], py[NP], pz[NP], td[NP];
    unsigned key[NP * 2];
#pragma unroll
    for (int j = 0; j < NP * 2; ++j) {
        const int slot = t + T * (j / R);
        const int k = slot + 512 * (j % R);
        const bool ok = (j < PPT) && (k < n);
        const float x = ok ? sxyz[k * 3 + 0] : 0.f, y = ok ? sxyz[k * 3 + 1] : 0.f, z = ok ? sxyz[k * 3 + 2] : 0.f;
        const float d0 = ok ? 1e38f : -1.f;        // tf_sampling_g.cu:118 ; -1 never beats best=-1 and fminf keeps it
        key[j] = fps_tie_key(ok ? k : 0);
        if (j & 1) { px[j / 2].y = x; py[j / 2].y = y; pz[j / 2].y = z; td[j / 2].y = d0; }
        else       { px[j / 2].x = x; py[j / 2].x = y; pz[j / 2].x = z; td[j / 2].x = d0; }
    }

    int old = 0;                                                   // seed index 0 (tf_sampling_g.cu:114)
    if (t == 0) s_sel[0] = 0;
    for (int j = 1; j < m; ++j) {
        const float x1 = sxyz[old * 3 + 0], y1 = sxyz[old * 3 + 1], z1 = sxyz[old * 3 + 2];
        const float2 nx = make_float2(-x1, -x1), ny = make_float2(-y1, -y1), nz = make_float2(-z1, -z1);
        float best = -1.f;
        unsigned bkey = 0xffffffffu;
#pragma unroll
        for (int q = 0; q < NP; ++q) {
            // FMUL dy*dy ; FFMA dx,dx ; FFMA dz,dz : per element the reference's contraction, two points per float pair
            const float2 dx = fadd2_rn(px[q], nx), dy = fadd2_rn(py[q], ny), dz = fadd2_rn(pz[q], nz);
            float2 d = fmul2_rn(dy, dy);
            d = ffma2_rn(dx, dx, d);
            d = ffma2_rn(dz, dz, d);
            td[q].x = fminf(d.x, td[q].x);                         // NaN d leaves td unchanged, as CUDA min() does
            td[q].y = fminf(d.y, td[q].y);
            if (td[q].x > best) { best = td[q].x; bkey = key[2 * q]; }
            if (td[q].y > best) { best = td[q].y; bkey = key[2 * q + 1]; }
        }
        // best is -1 or a non-negative float (incl. +inf): signed-int order == float order
        const int v = __float_as_int(best);
        const int wmax = __reduce_max_sync(0xffffffffu, v);
        const unsigned wkey = __reduce_min_sync(0xffffffffu, v == wmax ? bkey : 0xffffffffu);
        const int par = j & 1;
        if (lane == 0) { s_wval[par][warp] = wmax; s_wkey[par][warp] = wkey; }
        __syncthreads();
        const int pv = (lane < W) ? s_wval[par][lane] : INT_MIN;
        const unsigned pk = (lane < W) ? s_wkey[par][lane] : 0xffffffffu;
        const int gmax = __reduce_max_sync(0xffffffffu, pv);
        const unsigned gkey = __reduce_min_sync(0xffffffffu, pv == gmax ? pk : 0xffffffffu);
        old = gkey == 0xffffffffu ? 0 : fps_key_to_index(gkey);   // all-invalid cannot happen for n >= 1
        if (t == 0) s_sel[j] = old;
    }
    __syncthreads();
    int* io = idx_out + (size_t)cloud * m;
    for (int j = t; j < m; j += T) io[j] = s_sel[j];
    if (new_xyz != nullptr) {
        float* o = new_xyz + (size_t)cloud * m * 3;
        for (int e = t; e < m * 3; e += T) {
            int j = e / 3, c = e - j * 3;
            o[e] = sxyz[s_sel[j] * 3 + c];
        }
    }
}

__global__ void gather_point_kernel(int n, int m, long long total, const float* __restrict__ inp,
                                    const int* __restrict__ idx, float* __restrict__ out) {
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        long long row = e / 3;
        int c = (int)(e - row * 3);
        long long bi = row / m;
        int a = idx[row];
        out[e] = inp[(bi * n + a) * 3 + c];
    }
}

template <int T, int R>
static int launch_fps(int b, int n, int m, const float* xyz, int* idx, float* new_xyz, cudaStream_t st) {
    size_t smem = (size_t)n * 3 * sizeof(float) + (size_t)m * sizeof(int);
    PSA_SUPPORTED(smem <= 200 * 1024, "farthest_point_sample: n=%d, m=%d needs %zu B of shared memory", n, m, smem);
    PSA_CUDA(cudaFuncSetAttribute(fps_kernel<T, R>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    fps_kernel<T, R><<<b, T, smem, st>>>(n, m, xyz, idx, new_xyz);
    return check_launch("fps_kernel");
}

static inline int grid_for(long long total, int block) {
    long long g = (total + block - 1) / block;
    long long cap = (long long)kNumSMs * 16;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace psa

using namespace psa;

extern "C" int psa_farthest_point_sample(int b, int n, int m, const float* xyz, int* idx, float* new_xyz,
                                         psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 0 && m >= 0, "FarthestPointSample: negative dimension (b=%d n=%d m=%d)", b, n, m);
    if (b == 0 || m == 0) return PSA_OK;
    PSA_REQUIRE(n >= 1, "FarthestPointSample expects at least one input point (n=%d)", n);
    PSA_REQUIRE(xyz != nullptr && idx != nullptr, "FarthestPointSample: null buffer");
    cudaStream_t st = as_stream(stream);
    const int r = (n + 511) / 512;      // points per reference slot
    if (r <= 1) return launch_fps<128, 1>(b, n, m, xyz, idx, new_xyz, st);
    if (r <= 2) return launch_fps<128, 2>(b, n, m, xyz, idx, new_xyz, st);
    if (r <= 4) return launch_fps<128, 4>(b, n, m, xyz, idx, new_xyz, st);
    if (r <= 8) return launch_fps<256, 8>(b, n, m, xyz, idx, new_xyz, st);
    if (r <= 16) return launch_fps<512, 16>(b, n, m, xyz, idx, new_xyz, st);
    PSA_SUPPORTED(false, "farthest_point_sample: n=%d exceeds the register-resident limit of %d points", n, 16 * 512);
}

extern "C" int psa_gather_point(int b, int n, int m, const float* inp, const int* idx, float* out,
                                psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 0 && m >= 0, "GatherPoint: negative dimension");
    long long total = (long long)b * m * 3;
    if (total == 0) return PSA_OK;
    PSA_REQUIRE(inp && idx && out, "GatherPoint: null buffer");
    gather_point_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(n, m, total, inp, idx, out);
    return check_launch("gather_point_kernel");
}

