// pointcnn_train.cu -- PointCNN's X-Conv layer in training mode (PointCNN/pointcnn.py:10-52, pointfly.py:298-347 with
// is_training=True): the forward's batch-statistics stages and the backward of the core (psa_xconv_core, pointcnn.cu).
//
// Forward.  Batch norm needs each layer's whole batch before the next layer can run, so the core's stages are split at every batch
// norm.  Each stage kernel saves a = elu(z) (z for X_2, which has no ELU), the one tensor a batch-norm-after-ELU layer needs; the
// next stage applies the batch's (s, t) to a in registers.  Every pre-batch-norm value z is evaluated with xconv_core_kernel's own
// fmaf chain (same operands, same order, same elu), so psa_xconv_core run with the batch (s, t) computes its depthwise output from
// exactly the saved activations.
//   stage 0   local (R*K, 3) = pts[idx] - q;  a_p0 (R*K, C_pts) = elu(local . W_p0);  a_x0 (R, K*K) = elu(local (3K) . W_x0)
//   stage 1   a_p1 = elu(BN(a_p0) . W_p1);  a_x1 = elu(depthwise(BN(a_x0), W_x1))
//   stage 2   a_x2 = depthwise(BN(a_x1), W_x2)
// R = b*P queries.  Batch statistics between stages come from psa_bn_finalize_rows.
//
// Backward, fp32 FMA, no float atomics: weight gradients are summed per block over a fixed set of tiles (a grid that depends on the
// shape only) and the block partials added in block order (reduce_partials), so a step is bit-reproducible.
//   xconv_bwd_top_kernel     from d dw: fts_X = X2n . F recomputed, d fts_X = d dw . W_dw^T, dX2n = d fts_X . F^T,
//                            dF = X2n^T . d fts_X (split into the lifted columns and the gathered previous features), dW_dw
//   xconv_dw_bwd_kernel      a depthwise layer z[b*K + m] = sum_a x[a*K + b] W[a][b][m]: dW and dx from dz = the batch-norm
//                            backward of the layer (psa_grad_in) times the ELU gradient of its output
//   elu_bn_dy_kernel         the same dz materialised for the dense products (train_gemm.cuh)
//   bn_affine_rows_kernel    h = a * s + t through a row stride (a layer's slice of a wider output row)
#include "train_gemm.cuh"

namespace psa {

constexpr int kPtThreads = 256;
constexpr int kPtMaxK = 16;                    // psa_xconv_core's limit
constexpr int kPtSmemBudget = 200 * 1024;
constexpr int kPtMaxBlocks = 2 * kNumSMs;      // blocks of the weight-gradient kernels: partials = this many copies at most

// pointcnn.cu's elu: the stage kernels must round exactly as xconv_core_kernel does
__device__ __forceinline__ float pcnn_elu(float x) { return x > 0.f ? x : expm1f(x); }

// TF's EluGrad on the output a = elu(z): dz = g * (a + 1) where a < 0, g elsewhere
__device__ __forceinline__ float elu_grad(float g, float a) { return a < 0.f ? g * (a + 1.f) : g; }

struct PtStage {
    long long rows;              // b * P
    int n, P, K, Cf;
    const float* pts;
    const float* qrs;
    const int* idx;
    psa_xconv w;
    psa_xconv_saved s;
};

__device__ __forceinline__ float local_coord(const PtStage& a, long long r, int j, int dd) {
    const long long b = r / a.P;
    const int nb = __ldg(a.idx + r * a.K + j);
    return __fsub_rn(__ldg(a.pts + ((size_t)b * a.n + nb) * 3 + dd), __ldg(a.qrs + (size_t)r * 3 + dd));
}

__global__ void __launch_bounds__(kPtThreads) xconv_stage0_kernel(const __grid_constant__ PtStage a) {
    const int K = a.K, Cf = a.Cf, KK = K * K;
    const long long nl = a.rows * K * 3, np = a.rows * K * Cf, nx = a.rows * KK;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < nl + np + nx; e += (long long)gridDim.x * blockDim.x) {
        if (e < nl) {
            const long long rk = e / 3;
            a.s.local[e] = local_coord(a, rk / K, (int)(rk % K), (int)(e - rk * 3));
        } else if (e < nl + np) {
            const long long f = e - nl, rk = f / Cf;
            const int c = (int)(f - rk * Cf);
            const long long r = rk / K;
            const int j = (int)(rk - r * K);
            float s = 0.f;
#pragma unroll
            for (int dd = 0; dd < 3; ++dd) s = fmaf(local_coord(a, r, j, dd), __ldg(a.w.w_pts0 + dd * Cf + c), s);
            a.s.a_p0[f] = pcnn_elu(s);
        } else {
            const long long f = e - nl - np, r = f / KK;
            const int o = (int)(f - r * KK);
            float s = 0.f;
            for (int jd = 0; jd < 3 * K; ++jd) s = fmaf(local_coord(a, r, jd / 3, jd % 3), __ldg(a.w.w_x0 + (size_t)jd * KK + o), s);
            a.s.a_x0[f] = pcnn_elu(s);
        }
    }
}

// z[bb*K + mm] = sum_aa BN(x)[aa*K + bb] W[aa][bb][mm], the order of xconv_core_kernel's X1 / X2 loops
__device__ __forceinline__ float depthwise_z(const float* x, const float* s, const float* t, const float* W, int K, int o) {
    const int bb = o / K, mm = o - bb * K;
    float z = 0.f;
    for (int aa = 0; aa < K; ++aa) {
        const int i = aa * K + bb;
        z = fmaf(fmaf(__ldg(x + i), __ldg(s + i), __ldg(t + i)), __ldg(W + i * K + mm), z);
    }
    return z;
}

__global__ void __launch_bounds__(kPtThreads) xconv_stage1_kernel(const __grid_constant__ PtStage a) {
    const int K = a.K, Cf = a.Cf, KK = K * K;
    const long long np = a.rows * K * Cf, nx = a.rows * KK;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < np + nx; e += (long long)gridDim.x * blockDim.x) {
        if (e < np) {
            const long long rk = e / Cf;
            const int c = (int)(e - rk * Cf);
            const float* h = a.s.a_p0 + rk * Cf;
            float s = 0.f;
            for (int i = 0; i < Cf; ++i) s = fmaf(fmaf(__ldg(h + i), __ldg(a.w.s_pts0 + i), __ldg(a.w.t_pts0 + i)), __ldg(a.w.w_pts1 + i * Cf + c), s);
            a.s.a_p1[e] = pcnn_elu(s);
        } else {
            const long long f = e - np, r = f / KK;
            a.s.a_x1[f] = pcnn_elu(depthwise_z(a.s.a_x0 + r * KK, a.w.s_x0, a.w.t_x0, a.w.w_x1, K, (int)(f - r * KK)));
        }
    }
}

__global__ void __launch_bounds__(kPtThreads) xconv_stage2_kernel(const __grid_constant__ PtStage a) {
    const int K = a.K, KK = K * K;
    for (long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x; f < a.rows * KK; f += (long long)gridDim.x * blockDim.x) {
        const long long r = f / KK;
        a.s.a_x2[f] = depthwise_z(a.s.a_x1 + r * KK, a.w.s_x1, a.w.t_x1, a.w.w_x2, K, (int)(f - r * KK));
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Backward of the core's top: fts_X, the depthwise stage, X2 . F.  Block = tiles t = blockIdx.x, + gridDim.x, ... of QT queries;
// per query in shared memory X2n (K*K), F (K, Cin) and T (K, Cin) = fts_X, then d fts_X; the block's dW_dw sum in `acc`.
// ------------------------------------------------------------------------------------------------------------------
struct PtTop {
    long long rows;
    int n, P, K, Cf, Cp, Cin, dm, QT;
    const int* idx;
    const float* fts;            // (b*n, Cp) or null
    psa_xconv w;
    const float* a_p1;           // (R*K, Cf)
    const float* a_x2;           // (R, K*K)
    const float* d_dw;           // (R, Cin*dm)
    float* dX2n;                 // (R, K*K)
    float* dF_lift;              // (R*K, Cf)
    float* dF_prev;              // (R*K, Cp) or null
    float* partial;              // (gridDim.x, K*Cin*dm)
};

__host__ __device__ inline int top_query_floats(int K, int Cin) { return K * K + 2 * K * Cin; }

__global__ void __launch_bounds__(kPtThreads) xconv_bwd_top_kernel(const __grid_constant__ PtTop a) {
    extern __shared__ float s_t[];
    const int tid = threadIdx.x, QT = a.QT, K = a.K, Cf = a.Cf, Cin = a.Cin, dm = a.dm, KK = K * K;
    const int nw = K * Cin * dm, per = top_query_floats(K, Cin);
    float* acc = s_t;
    // query q's region: X2 (K*K) | F (K, Cin) | T (K, Cin)
#define X2(q) (s_t + nw + (q) * per)
#define F(q) (s_t + nw + (q) * per + KK)
#define T(q) (s_t + nw + (q) * per + KK + K * Cin)
    for (int e = tid; e < nw; e += kPtThreads) acc[e] = 0.f;
    const long long tiles = (a.rows + QT - 1) / QT;
    for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const long long r0 = tile * QT;
        const int nq = (int)min((long long)QT, a.rows - r0);
        for (int e = tid; e < QT * KK; e += kPtThreads) {
            const int q = e % QT, o = e / QT;
            if (q < nq) X2(q)[o] = fmaf(__ldg(a.a_x2 + (r0 + q) * KK + o), __ldg(a.w.s_x2 + o), __ldg(a.w.t_x2 + o));
        }
        for (int e = tid; e < QT * K * Cin; e += kPtThreads) {
            const int q = e % QT, jc = e / QT, j = jc / Cin, c = jc - j * Cin;
            if (q >= nq) continue;
            const long long r = r0 + q;
            float v;
            if (c < Cf) {
                v = fmaf(__ldg(a.a_p1 + (r * K + j) * Cf + c), __ldg(a.w.s_pts1 + c), __ldg(a.w.t_pts1 + c));
            } else {
                const long long b = r / a.P;
                v = __ldg(a.fts + ((size_t)b * a.n + __ldg(a.idx + r * K + j)) * a.Cp + (c - Cf));
            }
            F(q)[jc] = v;
        }
        __syncthreads();
        // fts_X[i][c] = sum_j X2[i][j] F[j][c]
        for (int e = tid; e < QT * K * Cin; e += kPtThreads) {
            const int q = e % QT, ic = e / QT, i = ic / Cin, c = ic - i * Cin;
            if (q >= nq) continue;
            const float* x2 = X2(q) + i * K;
            const float* f = F(q) + c;
            float s = 0.f;
            for (int j = 0; j < K; ++j) s = fmaf(x2[j], f[j * Cin], s);
            T(q)[ic] = s;
        }
        __syncthreads();
        // dW_dw[i][c][m] += sum over the tile's queries, in query order
        for (int e = tid; e < nw; e += kPtThreads) {
            const int m = e % dm, ic = e / dm, c = ic % Cin;
            float s = acc[e];
            for (int q = 0; q < nq; ++q) s = fmaf(T(q)[ic], __ldg(a.d_dw + (r0 + q) * Cin * dm + c * dm + m), s);
            acc[e] = s;
        }
        __syncthreads();
        // d fts_X[i][c] = sum_m d dw[c*dm + m] W_dw[i][c][m]
        for (int e = tid; e < QT * K * Cin; e += kPtThreads) {
            const int q = e % QT, ic = e / QT, c = ic % Cin;
            if (q >= nq) continue;
            const float* g = a.d_dw + (r0 + q) * Cin * dm + c * dm;
            const float* w = a.w.w_dw + (size_t)ic * dm;
            float s = 0.f;
            for (int m = 0; m < dm; ++m) s = fmaf(__ldg(g + m), __ldg(w + m), s);
            T(q)[ic] = s;
        }
        __syncthreads();
        // dX2n[i][j] = sum_c dT[i][c] F[j][c];  dF[j][c] = sum_i X2[i][j] dT[i][c]
        for (int e = tid; e < QT * KK; e += kPtThreads) {
            const int q = e % QT, o = e / QT, i = o / K, j = o - i * K;
            if (q >= nq) continue;
            const float* t = T(q) + i * Cin;
            const float* f = F(q) + j * Cin;
            float s = 0.f;
            for (int c = 0; c < Cin; ++c) s = fmaf(t[c], f[c], s);
            a.dX2n[(r0 + q) * KK + o] = s;
        }
        for (int e = tid; e < QT * K * Cin; e += kPtThreads) {
            const int q = e % QT, jc = e / QT, j = jc / Cin, c = jc - j * Cin;
            if (q >= nq) continue;
            const float* x2 = X2(q) + j;
            const float* t = T(q) + c;
            float s = 0.f;
            for (int i = 0; i < K; ++i) s = fmaf(x2[i * K], t[i * Cin], s);
            const long long rk = (r0 + q) * K + j;
            if (c < Cf) a.dF_lift[rk * Cf + c] = s;
            else a.dF_prev[rk * a.Cp + (c - Cf)] = s;
        }
        __syncthreads();
    }
    for (int e = tid; e < nw; e += kPtThreads) a.partial[(size_t)blockIdx.x * nw + e] = acc[e];
#undef X2
#undef F
#undef T
}

// ------------------------------------------------------------------------------------------------------------------
// Backward of a depthwise X layer z[bb*K + mm] = sum_aa x[aa*K + bb] W[aa][bb][mm], x = BN(a_in):
//   dW[aa][bb][mm] = sum_r x[aa*K + bb] dz[bb*K + mm],  dx[aa*K + bb] = sum_mm dz[bb*K + mm] W[aa][bb][mm]
// dz = g (the batch-norm backward of the layer's output) times the ELU gradient when `elu`.  Tiles of QT queries as above.
// ------------------------------------------------------------------------------------------------------------------
struct PtDw {
    long long rows;
    int K, QT, elu;
    const float* x;              // (R, K*K) saved activations of the input layer
    const float* s;              // its batch (s, t)
    const float* t;
    GradIn g;                    // over (R, K*K): y = this layer's saved activations
    const float* W;              // (K, K, K)
    float* dx;                   // (R, K*K): the gradient of BN(a_in)
    float* partial;              // (gridDim.x, K^3)
};

__device__ __forceinline__ float gated(const GradIn& g, int elu, long long r, int c) {
    const float v = g.get(r, c);
    return elu ? elu_grad(v, __ldg(g.y + r * g.ld + c)) : v;
}

__global__ void __launch_bounds__(kPtThreads) xconv_dw_bwd_kernel(const __grid_constant__ PtDw a) {
    extern __shared__ float s_d[];
    const int tid = threadIdx.x, QT = a.QT, K = a.K, KK = K * K, nw = KK * K;
    float* acc = s_d;
    float* X = s_d + nw;                     // (KK, QT): element o of query q at o * QT + q
    float* G = X + KK * QT;
    for (int e = tid; e < nw; e += kPtThreads) acc[e] = 0.f;
    const long long tiles = (a.rows + QT - 1) / QT;
    for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const long long r0 = tile * QT;
        const int nq = (int)min((long long)QT, a.rows - r0);
        for (int e = tid; e < QT * KK; e += kPtThreads) {
            const int q = e % QT, o = e / QT;
            if (q >= nq) continue;
            const long long r = r0 + q;
            X[e] = fmaf(__ldg(a.x + r * KK + o), __ldg(a.s + o), __ldg(a.t + o));
            G[e] = gated(a.g, a.elu, r, o);
        }
        __syncthreads();
        for (int e = tid; e < nw; e += kPtThreads) {
            const int i = e / K, bb = i % K, mm = e - i * K;       // i = aa*K + bb
            const float* x = X + i * QT;
            const float* g = G + (bb * K + mm) * QT;
            float s = acc[e];
            for (int q = 0; q < nq; ++q) s = fmaf(x[q], g[q], s);
            acc[e] = s;
        }
        for (int e = tid; e < QT * KK; e += kPtThreads) {
            const int q = e % QT, i = e / QT, bb = i % K;
            if (q >= nq) continue;
            const float* w = a.W + (size_t)i * K;
            float s = 0.f;
            for (int mm = 0; mm < K; ++mm) s = fmaf(G[(bb * K + mm) * QT + q], __ldg(w + mm), s);
            a.dx[(r0 + q) * KK + i] = s;
        }
        __syncthreads();
    }
    for (int e = tid; e < nw; e += kPtThreads) a.partial[(size_t)blockIdx.x * nw + e] = acc[e];
}

__global__ void elu_bn_dy_kernel(long long rows, int C, const GradIn g, float* __restrict__ dz) {
    const long long total = rows * C;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const long long r = e / C;
        dz[e] = gated(g, 1, r, (int)(e - r * C));
    }
}

__global__ void bn_affine_rows_kernel(long long rows, int C, const float* __restrict__ a, const float* __restrict__ s,
                                      const float* __restrict__ t, float* __restrict__ out, long long ldo) {
    const long long total = rows * C;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const long long r = e / C;
        const int c = (int)(e - r * C);
        out[r * ldo + c] = fmaf(__ldg(a + e), __ldg(s + c), __ldg(t + c));
    }
}

static unsigned pt_grid(long long total) {
    const long long g = (total + kPtThreads - 1) / kPtThreads;
    return (unsigned)(g < 1 ? 1 : g > 16 * kNumSMs ? 16 * kNumSMs : g);
}

static int top_qt(int K, int Cin, int dm) {
    const long long free_floats = kPtSmemBudget / 4 - (long long)K * Cin * dm;
    const long long q = free_floats / top_query_floats(K, Cin);
    return (int)(q < 16 ? q : 16);
}
static int top_blocks(long long rows, int qt) {
    const long long tiles = (rows + qt - 1) / qt;
    return (int)(tiles < kPtMaxBlocks ? tiles : kPtMaxBlocks);
}
constexpr int kDwQT = 32;
static int dw_blocks(long long rows) {
    const long long tiles = (rows + kDwQT - 1) / kDwQT;
    return (int)(tiles < kPtMaxBlocks ? tiles : kPtMaxBlocks);
}

}  // namespace psa

using namespace psa;

static int xconv_dims_ok(const char* fn, int b, int n, int P, const psa_xconv* w) {
    PSA_REQUIRE(w != nullptr, "%s: null layer", fn);
    PSA_REQUIRE(b >= 0 && n >= 1 && P >= 1, "%s: bad dims b=%d n=%d P=%d", fn, b, n, P);
    PSA_REQUIRE(w->K >= 1 && w->K <= kPtMaxK && w->K <= n, "%s: K=%d must be in [1, min(%d, n=%d)]", fn, w->K, kPtMaxK, n);
    PSA_REQUIRE(w->c_pts >= 1 && w->c_prev >= 0 && w->dm >= 1, "%s: bad widths c_pts=%d c_prev=%d dm=%d", fn, w->c_pts, w->c_prev, w->dm);
    return PSA_OK;
}

extern "C" int psa_xconv_train_stage(int stage, int b, int n, int P, const float* pts, const float* qrs, const int* idx, const psa_xconv* layer,
                                     const psa_xconv_saved* saved, psa_stream_t stream) {
    PSA_REQUIRE(stage >= 0 && stage <= 2, "xconv_train_stage: stage %d (0, 1 or 2)", stage);
    int rc = xconv_dims_ok("xconv_train_stage", b, n, P, layer);
    if (rc != PSA_OK) return rc;
    PSA_REQUIRE(saved != nullptr, "xconv_train_stage: null saved");
    if (b == 0) return PSA_OK;
    const psa_xconv& w = *layer;
    const psa_xconv_saved& s = *saved;
    PtStage a;
    a.rows = (long long)b * P; a.n = n; a.P = P; a.K = w.K; a.Cf = w.c_pts; a.pts = pts; a.qrs = qrs; a.idx = idx; a.w = w; a.s = s;
    const long long R = a.rows, RK = R * w.K, KK = (long long)w.K * w.K;
    cudaStream_t st = as_stream(stream);
    if (stage == 0) {
        PSA_REQUIRE(pts && qrs && idx && w.w_pts0 && w.w_x0 && s.local && s.a_p0 && s.a_x0, "xconv_train_stage: null buffer");
        xconv_stage0_kernel<<<pt_grid(RK * 3 + RK * w.c_pts + R * KK), kPtThreads, 0, st>>>(a);
        return check_launch("xconv_stage0_kernel");
    }
    if (stage == 1) {
        PSA_REQUIRE(w.w_pts1 && w.s_pts0 && w.t_pts0 && w.w_x1 && w.s_x0 && w.t_x0 && s.a_p0 && s.a_x0 && s.a_p1 && s.a_x1,
                    "xconv_train_stage: null buffer");
        xconv_stage1_kernel<<<pt_grid(RK * w.c_pts + R * KK), kPtThreads, 0, st>>>(a);
        return check_launch("xconv_stage1_kernel");
    }
    PSA_REQUIRE(w.w_x2 && w.s_x1 && w.t_x1 && s.a_x1 && s.a_x2, "xconv_train_stage: null buffer");
    xconv_stage2_kernel<<<pt_grid(R * KK), kPtThreads, 0, st>>>(a);
    return check_launch("xconv_stage2_kernel");
}

extern "C" size_t psa_xconv_train_bwd_workspace_bytes(int b, int P, int K, int c_pts, int c_prev, int dm) {
    if (b < 1 || P < 1 || K < 1 || K > kPtMaxK || c_pts < 1 || c_prev < 0 || dm < 1) return 0;
    const long long rows = (long long)b * P;
    const int Cin = c_pts + c_prev, qt = top_qt(K, Cin, dm);
    if (qt < 1) return 0;
    const size_t top = (size_t)top_blocks(rows, qt) * K * Cin * dm * sizeof(float);
    const size_t dw = (size_t)dw_blocks(rows) * K * K * K * sizeof(float);
    return top > dw ? top : dw;
}

extern "C" int psa_xconv_train_bwd_top(int b, int n, int P, const int* idx, const float* fts, const psa_xconv* layer, const psa_xconv_saved* saved,
                                       const float* d_dw, float* dX2n, float* dF_lift, float* dF_prev, float* dW_dw, void* workspace,
                                       size_t workspace_bytes, psa_stream_t stream) {
    int rc = xconv_dims_ok("xconv_train_bwd_top", b, n, P, layer);
    if (rc != PSA_OK) return rc;
    const psa_xconv& w = *layer;
    PSA_REQUIRE((w.c_prev == 0) == (fts == nullptr) && (w.c_prev == 0) == (dF_prev == nullptr),
                "xconv_train_bwd_top: fts and dF_prev are given exactly when c_prev > 0");
    const int Cin = w.c_pts + w.c_prev, qt = top_qt(w.K, Cin, w.dm);
    PSA_SUPPORTED(qt >= 1, "xconv_train_bwd_top: K=%d, C_in=%d, dm=%d exceed the shared-memory budget", w.K, Cin, w.dm);
    if (b == 0) return PSA_OK;
    PSA_REQUIRE(saved && idx && d_dw && dX2n && dF_lift && dW_dw && saved->a_p1 && saved->a_x2 && w.s_pts1 && w.t_pts1 && w.s_x2 && w.t_x2 && w.w_dw,
                "xconv_train_bwd_top: null buffer");
    const size_t need = psa_xconv_train_bwd_workspace_bytes(b, P, w.K, w.c_pts, w.c_prev, w.dm);
    PSA_REQUIRE(workspace && workspace_bytes >= need, "xconv_train_bwd_top: workspace of %zu bytes required, got %zu", need, workspace_bytes);
    PtTop a;
    a.rows = (long long)b * P; a.n = n; a.P = P; a.K = w.K; a.Cf = w.c_pts; a.Cp = w.c_prev; a.Cin = Cin; a.dm = w.dm; a.QT = qt;
    a.idx = idx; a.fts = fts; a.w = w; a.a_p1 = saved->a_p1; a.a_x2 = saved->a_x2; a.d_dw = d_dw; a.dX2n = dX2n; a.dF_lift = dF_lift;
    a.dF_prev = dF_prev; a.partial = reinterpret_cast<float*>(workspace);
    const int blocks = top_blocks(a.rows, qt);
    const size_t smem = ((size_t)w.K * Cin * w.dm + (size_t)qt * top_query_floats(w.K, Cin)) * sizeof(float);
    cudaStream_t st = as_stream(stream);
    PSA_CUDA(cudaFuncSetAttribute(xconv_bwd_top_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    xconv_bwd_top_kernel<<<blocks, kPtThreads, smem, st>>>(a);
    rc = check_launch("xconv_bwd_top_kernel");
    if (rc != PSA_OK) return rc;
    return reduce_partials(blocks, w.K * Cin * w.dm, a.partial, dW_dw, st);
}

extern "C" int psa_xconv_depthwise_bwd(long long rows, int K, const float* x, const float* s, const float* t, const psa_grad_in* g, int elu,
                                       const float* W, float* dW, float* dx, void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    PSA_REQUIRE(rows >= 0 && K >= 1 && K <= kPtMaxK, "xconv_depthwise_bwd: bad dims rows=%lld K=%d", rows, K);
    PSA_REQUIRE(g != nullptr && g->mode == 0, "xconv_depthwise_bwd: a mode-0 psa_grad_in is required");
    if (rows == 0) return PSA_OK;
    PSA_REQUIRE(x && s && t && W && dW && dx && g->dh && g->y, "xconv_depthwise_bwd: null buffer");
    const size_t need = (size_t)dw_blocks(rows) * K * K * K * sizeof(float);
    PSA_REQUIRE(workspace && workspace_bytes >= need, "xconv_depthwise_bwd: workspace of %zu bytes required, got %zu", need, workspace_bytes);
    PtDw a;
    a.rows = rows; a.K = K; a.QT = kDwQT; a.elu = elu != 0; a.x = x; a.s = s; a.t = t; a.g = GradIn(*g); a.W = W; a.dx = dx;
    a.partial = reinterpret_cast<float*>(workspace);
    const int blocks = dw_blocks(rows);
    const size_t smem = ((size_t)K * K * K + 2 * (size_t)kDwQT * K * K) * sizeof(float);
    cudaStream_t st = as_stream(stream);
    PSA_CUDA(cudaFuncSetAttribute(xconv_dw_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    xconv_dw_bwd_kernel<<<blocks, kPtThreads, smem, st>>>(a);
    const int rc = check_launch("xconv_dw_bwd_kernel");
    if (rc != PSA_OK) return rc;
    return reduce_partials(blocks, K * K * K, a.partial, dW, st);
}

extern "C" int psa_elu_bn_dy(long long rows, int C, const psa_grad_in* g, float* dz, psa_stream_t stream) {
    PSA_REQUIRE(rows >= 0 && C >= 1, "elu_bn_dy: bad dims rows=%lld C=%d", rows, C);
    PSA_REQUIRE(g != nullptr && g->mode == 0, "elu_bn_dy: a mode-0 psa_grad_in is required");
    if (rows == 0) return PSA_OK;
    PSA_REQUIRE(g->dh && g->y && dz, "elu_bn_dy: null buffer");
    elu_bn_dy_kernel<<<pt_grid(rows * C), kPtThreads, 0, as_stream(stream)>>>(rows, C, GradIn(*g), dz);
    return check_launch("elu_bn_dy_kernel");
}

extern "C" int psa_bn_affine_rows(long long rows, int C, const float* a, const float* s, const float* t, float* out, long long ldo,
                                  psa_stream_t stream) {
    PSA_REQUIRE(rows >= 0 && C >= 1 && ldo >= C, "bn_affine_rows: bad dims rows=%lld C=%d ldo=%lld", rows, C, ldo);
    if (rows == 0) return PSA_OK;
    PSA_REQUIRE(a && s && t && out, "bn_affine_rows: null buffer");
    bn_affine_rows_kernel<<<pt_grid(rows * C), kPtThreads, 0, as_stream(stream)>>>(rows, C, a, s, t, out, ldo);
    return check_launch("bn_affine_rows_kernel");
}
