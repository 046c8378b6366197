// mfv_train.cu -- 3DmFV-Net's training backward (3DmFV-Net/models/3dmfv_net_cls.py:29-102, utils/tf_util.py:254-311 conv3d,
// :406-429 pools, :458-495 batch norm): the two products of every SAME, stride-1 conv3d, the batch-norm pieces the products read,
// and the pools' winners and backward.  The forward's convolutions are psa_conv3d_infer (mfv.cu).  fp32 FMA in every arithmetic
// mode (train_gemm.cuh explains why fp32 FMA holds the 1e-4 gradient bound without an operand split); no float atomics, every sum
// in a fixed order, so a step is bit-reproducible.
//
// Rows are voxel-major (row = voxel * b + cloud, voxel = (z * r + y) * r + x), K = k^3 * c in (tap, channel) order, tap =
// (dz * k + dy) * k + dx with offset (dz, dy, dx) - k / 2.  With dy (rows, c_out) the gradient of a conv's pre-batch-norm output:
//   weight gradient  dW[(tap, ch)][o] = sum_rows x[row + offset(tap)][ch] * dy[row][o]      train_gemm_kernel, A = MfvConvA
//                    (the conv input gathered as psa_conv3d_infer's FMA kernel reads it, transposed), split over the rows
//   data gradient    dx[u][ch] = sum_(tap, o) dy[u - offset(tap)][o] * W[(tap, ch)][o]       train_gemm_kernel, A = MfvGradA,
//                    B = MfvWt (W read transposed), split over the taps, partials added in split order by mfv_grad_finish_kernel
// Neither forms the (rows, K) im2col operand.  Tap skipping (GemmSkipK): a 16-wide contraction block is skipped when, for every
// tap it involves, the tap lies outside the grid for every row it involves -- the weight gradient asks it of a block of 16 rows
// and the 1-2 taps of a 128-row tile of dW, the data gradient of a tap and the rows of a 128-row tile of dx.  At b = 3 a block
// or a tile straddles voxels: the rule takes the first row at or after the block's start whose shifted voxel is inside the grid
// (mfv_first_row_in), so it is exact at any b.  A skipped block holds only zero products: skipping never changes a bit.
#include "train_gemm.cuh"

namespace psa {

constexpr long long kNoRow = 1LL << 62;

// the first row >= R whose voxel shifted by (oz, oy, ox) lies inside the r^3 grid, or kNoRow
__host__ __device__ inline long long mfv_first_row_in(long long R, int b, int r, int oz, int oy, int ox) {
    const int zl = oz < 0 ? -oz : 0, zh = oz > 0 ? r - oz : r, yl = oy < 0 ? -oy : 0, yh = oy > 0 ? r - oy : r;
    const int xl = ox < 0 ? -ox : 0, xh = ox > 0 ? r - ox : r;
    const long long v = R / b;
    if (zl >= zh || yl >= yh || xl >= xh || v >= (long long)r * r * r) return kNoRow;
    int z = (int)(v / (r * r)), y = (int)(v / r % r), x = (int)(v % r);
    bool moved = true;
    if (z < zl) { z = zl; y = yl; x = xl; }
    else if (z >= zh) return kNoRow;
    else if (y < yl) { y = yl; x = xl; }
    else if (y >= yh) { if (++z >= zh) return kNoRow; y = yl; x = xl; }
    else if (x < xl) { x = xl; }
    else if (x >= xh) {
        x = xl;
        if (++y >= yh) { if (++z >= zh) return kNoRow; y = yl; }
    } else {
        moved = false;
    }
    return moved ? (((long long)z * r + y) * r + x) * b : R;
}

struct MfvConvGeom {
    long long rows;     // b * r^3
    int b, r, k;
    __host__ __device__ void offset(int tap, int& oz, int& oy, int& ox) const {
        const int h = k / 2;
        oz = tap / (k * k) - h; oy = tap / k % k - h; ox = tap % k - h;
    }
    // the row holding voxel(R) shifted by `sign` * offset(tap), same cloud, or -1 outside the grid
    __device__ __forceinline__ long long shifted(long long R, int tap, int sign) const {
        int oz, oy, ox;
        offset(tap, oz, oy, ox);
        const long long v = R / b;
        const int cl = (int)(R - v * b);
        const int z = (int)(v / (r * r)) + sign * oz, y = (int)(v / r % r) + sign * oy, x = (int)(v % r) + sign * ox;
        if (z < 0 || z >= r || y < 0 || y >= r || x < 0 || x >= r) return -1;
        return ((long long)(z * r + y) * r + x) * b + cl;
    }
};

// weight gradient's A, read transposed (row = contraction row R, col = (tap, ch)): the conv input psa_conv3d_infer gathers
struct MfvConvA {
    static constexpr bool kSkipK = true;
    MfvConvGeom g;
    const float* x;
    long long ldx;
    int c, K;
    __device__ __forceinline__ float get(long long R, int kk) const {
        const int tap = kk / c;
        const long long s = g.shifted(R, tap, 1);
        return s >= 0 ? __ldg(x + s * ldx + (kk - tap * c)) : 0.f;
    }
    // four channels of one tap (c % 4 == 0, kk % 4 == 0)
    __device__ __forceinline__ float4 get4(long long R, int kk) const {
        const int tap = kk / c;
        const long long s = g.shifted(R, tap, 1);
        return s >= 0 ? __ldg(reinterpret_cast<const float4*>(x + s * ldx + (kk - tap * c))) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __device__ __forceinline__ bool vec_ok() const {
        return (c & 3) == 0 && (ldx & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
    }
    // the rows are the contraction: the next 16-row block with a row inside the grid for one of the tile's taps
    __host__ __device__ long long next_k(long long k, long long k_end, long long m0, int bm) const {
        const int t0 = (int)(m0 / c), t1 = (int)((m0 + bm < K ? m0 + bm : K) - 1) / c;
        long long best = kNoRow;
        for (int t = t0; t <= t1; ++t) {
            int oz, oy, ox;
            g.offset(t, oz, oy, ox);
            const long long f = mfv_first_row_in(k, g.b, g.r, oz, oy, ox);
            best = f < best ? f : best;
        }
        return best >= k_end ? k_end : k + (best - k) / kGemmBK * kGemmBK;
    }
};

// data gradient's A (row = u, col = (tap, o)): dy at u's voxel shifted by -offset(tap)
struct MfvGradA {
    static constexpr bool kSkipK = true;
    MfvConvGeom g;
    const float* dy;
    int N, taps;        // c_out, k^3
    __device__ __forceinline__ float get(long long u, int kk) const {
        const int tap = kk / N;
        const long long s = g.shifted(u, tap, -1);
        return s >= 0 ? __ldg(dy + s * N + (kk - tap * N)) : 0.f;
    }
    __device__ __forceinline__ float4 get4(long long u, int kk) const {
        const int tap = kk / N;
        const long long s = g.shifted(u, tap, -1);
        return s >= 0 ? __ldg(reinterpret_cast<const float4*>(dy + s * N + (kk - tap * N))) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __device__ __forceinline__ bool vec_ok() const { return (N & 3) == 0 && (reinterpret_cast<uintptr_t>(dy) & 15) == 0; }
    // the taps are the contraction: the first tap at or after k's that reaches inside the grid from one of the tile's rows
    __host__ __device__ long long next_k(long long k, long long k_end, long long m0, int bm) const {
        const long long last = (m0 + bm < g.rows ? m0 + bm : g.rows) - 1;
        for (int t = (int)(k / N); t < taps && (long long)t * N < k_end; ++t) {
            int oz, oy, ox;
            g.offset(t, oz, oy, ox);
            if (mfv_first_row_in(m0, g.b, g.r, -oz, -oy, -ox) <= last) {
                const long long s = (long long)t * N;
                return s <= k ? k : k + (s - k) / kGemmBK * kGemmBK;
            }
        }
        return k_end;
    }
};

// data gradient's B, contraction-contiguous (row = ch, col = (tap, o)): W[(tap, ch)][o]
struct MfvWt {
    const float* W;
    int c, N;
    __device__ __forceinline__ float get(long long ch, int kk) const {
        const int tap = kk / N;
        return __ldg(W + ((long long)tap * c + ch) * N + (kk - tap * N));
    }
    __device__ __forceinline__ float4 get4(long long ch, int kk) const {
        const int tap = kk / N;
        return __ldg(reinterpret_cast<const float4*>(W + ((long long)tap * c + ch) * N + (kk - tap * N)));
    }
    __device__ __forceinline__ bool vec_ok() const { return (N & 3) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0; }
};

constexpr int kMfvBM = 128, kMfvBN = 64;     // 128 x 64 tiles: the gathered operands' index arithmetic fits two CTAs per SM

struct MfvBwdPlan {
    int wsplits, dsplits;
    long long wkps, dkps;
    size_t bytes;
};

// weight gradient: weight_grad_splits over the rows; data gradient: taps per split so that tiles * splits fill two waves, <= 16
static MfvBwdPlan mfv_bwd_plan(int b, int r, int k, int c, int c_out) {
    MfvBwdPlan p{};
    const long long rows = (long long)b * r * r * r, K = (long long)k * k * k * c;
    const int wt = (int)(((K + kMfvBM - 1) / kMfvBM) * ((c_out + kMfvBN - 1) / kMfvBN));
    p.wsplits = weight_grad_splits(rows, wt, &p.wkps);
    const long long dt = ((rows + kMfvBM - 1) / kMfvBM) * ((c + kMfvBN - 1) / kMfvBN);
    const int taps = k * k * k;
    long long want = (2LL * kNumSMs + dt - 1) / dt;
    want = want < 16 ? want : 16;
    want = want < taps ? want : taps;
    want = want < 1 ? 1 : want;
    const long long per = (taps + want - 1) / want;                  // taps per split
    p.dkps = (per * c_out + kGemmBK - 1) / kGemmBK * kGemmBK;
    const long long Kd = (long long)taps * c_out;
    p.dsplits = (int)((Kd + p.dkps - 1) / p.dkps);
    const size_t wb = p.wsplits > 1 ? (size_t)p.wsplits * K * c_out * sizeof(float) : 0;
    const size_t db = (size_t)p.dsplits * rows * c * sizeof(float);
    p.bytes = ((wb > db ? wb : db) + 255) & ~(size_t)255;
    return p;
}

// dx[row * ld + col] = (accumulate ? dx : 0) + sum_sp partial[sp][row][col], the partials in split order
__global__ void mfv_grad_finish_kernel(int splits, long long rows, int c, const float* __restrict__ partial, float* __restrict__ dx,
                                       long long ld, int accumulate) {
    const long long total = rows * c;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const long long row = e / c;
        float s = __ldg(partial + e);
        for (int sp = 1; sp < splits; ++sp) s += __ldg(partial + (size_t)sp * total + e);
        float* d = dx + row * ld + (e - row * c);
        *d = accumulate ? *d + s : s;
    }
}

__global__ void mfv_bn_relu_kernel(long long rows, int C, const float* __restrict__ y, const float* __restrict__ scale,
                                   const float* __restrict__ shift, float* __restrict__ out, long long ldo) {
    const long long total = rows * C;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const long long row = e / C;
        const int ch = (int)(e - row * C);
        out[row * ldo + ch] = fmaxf(fmaf(__ldg(y + e), __ldg(scale + ch), __ldg(shift + ch)), 0.f);
    }
}

__global__ void mfv_bn_dy_kernel(long long rows, int C, const GradIn g, float* __restrict__ dy) {
    const long long total = rows * C;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const long long row = e / C;
        dy[e] = g.get(row, (int)(e - row * C));
    }
}

// SAME 2^3 stride-2 max with its winner (first maximum in (dz, dy, dx) order; far-end padding cells are left out)
__global__ void mfv_maxpool_win_kernel(int b, int r, int c, const float* __restrict__ x, float* __restrict__ out,
                                       uint8_t* __restrict__ win) {
    const int ro = (r + 1) / 2;
    const long long total = (long long)b * ro * ro * ro * c;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int ch = (int)(e % c);
        const long long row = e / c, v = row / b;
        const int cl = (int)(row - v * b), z = (int)(v / (ro * ro)), y = (int)(v / ro % ro), xx = (int)(v % ro);
        float m = 0.f;
        int w = -1;
        for (int p = 0; p < 8; ++p) {
            const int Z = 2 * z + (p >> 2), Y = 2 * y + ((p >> 1) & 1), X = 2 * xx + (p & 1);
            if (Z >= r || Y >= r || X >= r) continue;
            const float val = __ldg(x + ((long long)((Z * r + Y) * r + X) * b + cl) * c + ch);
            if (w < 0 || val > m) { m = val; w = p; }
        }
        out[e] = m;
        win[e] = (uint8_t)w;
    }
}

// 2^3 max backward: every cell belongs to one window; it takes the window's gradient when it is the recorded winner
__global__ void mfv_maxpool_bwd_kernel(int b, int r, int c, const float* __restrict__ dout, const uint8_t* __restrict__ win,
                                       float* __restrict__ dx) {
    const int ro = (r + 1) / 2;
    const long long total = (long long)b * r * r * r * c;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int ch = (int)(e % c);
        const long long row = e / c, v = row / b;
        const int cl = (int)(row - v * b), z = (int)(v / (r * r)), y = (int)(v / r % r), xx = (int)(v % r);
        const long long o = ((long long)(((z >> 1) * ro + (y >> 1)) * ro + (xx >> 1)) * b + cl) * c + ch;
        const int p = (z & 1) * 4 + (y & 1) * 2 + (xx & 1);
        dx[e] = __ldg(win + o) == p ? __ldg(dout + o) : 0.f;
    }
}

__device__ __forceinline__ int avg_count(int r, int z, int y, int x) {
    auto span = [r](int t) { return (t + 1 < r ? t + 1 : r - 1) - (t > 0 ? t - 1 : 0) + 1; };
    return span(z) * span(y) * span(x);
}

// 3^3 stride-1 average backward as a gather: cell u adds dout[v] / count(v) over the in-grid windows v holding it, (dz, dy, dx) order
__global__ void mfv_avgpool_bwd_kernel(int b, int r, int c, const float* __restrict__ dout, float* __restrict__ dx) {
    const long long total = (long long)b * r * r * r * c;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int ch = (int)(e % c);
        const long long row = e / c, v = row / b;
        const int cl = (int)(row - v * b), z = (int)(v / (r * r)), y = (int)(v / r % r), xx = (int)(v % r);
        float s = 0.f;
        for (int dz = -1; dz <= 1; ++dz)
            for (int dy = -1; dy <= 1; ++dy)
                for (int dxx = -1; dxx <= 1; ++dxx) {
                    const int Z = z + dz, Y = y + dy, X = xx + dxx;
                    if (Z < 0 || Z >= r || Y < 0 || Y >= r || X < 0 || X >= r) continue;
                    s += __ldg(dout + ((long long)((Z * r + Y) * r + X) * b + cl) * c + ch) / (float)avg_count(r, Z, Y, X);
                }
        dx[e] = s;
    }
}

static unsigned grid_for(long long total) { return (unsigned)min((total + 255) / 256, 8192LL); }

static int mfv_bwd_dims(const char* what, int b, int r, int k, int c, int c_out) {
    PSA_REQUIRE(b >= 0 && r >= 1 && c >= 1 && c_out >= 1, "%s: bad dims b=%d r=%d c=%d c_out=%d", what, b, r, c, c_out);
    PSA_REQUIRE(k == 1 || k == 3 || k == 5, "%s: k=%d must be 1, 3 or 5", what, k);
    PSA_REQUIRE(r < 256 && (long long)b * r * r * r < (1LL << 31) && (long long)k * k * k * c <= (1LL << 30) &&
                    (long long)k * k * k * c_out <= (1LL << 30), "%s: too large", what);
    return PSA_OK;
}

static MfvConvGeom mfv_geom(int b, int r, int k) { return MfvConvGeom{(long long)b * r * r * r, b, r, k}; }

}  // namespace psa

using namespace psa;

extern "C" size_t psa_conv3d_bwd_workspace_bytes(int b, int r, int k, int c, int c_out) {
    if (b < 1 || r < 1 || r >= 256 || (k != 1 && k != 3 && k != 5) || c < 1 || c_out < 1) return 0;
    return mfv_bwd_plan(b, r, k, c, c_out).bytes;
}

extern "C" int psa_conv3d_bwd_weight(int b, int r, int k, int c, int c_out, const float* x, long long ldx, const float* dy, float* dW,
                                     void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    int rc = mfv_bwd_dims("conv3d_bwd_weight", b, r, k, c, c_out);
    if (rc != PSA_OK) return rc;
    PSA_REQUIRE(ldx >= c, "conv3d_bwd_weight: row stride ldx=%lld below the width %d", ldx, c);
    if (b == 0) return PSA_OK;
    PSA_REQUIRE(x && dy && dW, "conv3d_bwd_weight: null buffer");
    const MfvBwdPlan pl = mfv_bwd_plan(b, r, k, c, c_out);
    const long long rows = (long long)b * r * r * r, K = (long long)k * k * k * c;
    GemmOut o;
    o.ld_out = c_out; o.bias = nullptr; o.col_skip = 0; o.stat_partial = nullptr;
    o.out = dW;
    if (pl.wsplits > 1) {
        PSA_REQUIRE(workspace != nullptr && workspace_bytes >= pl.bytes,
                    "conv3d_bwd_weight: workspace of %zu bytes required (psa_conv3d_bwd_workspace_bytes), got %zu", pl.bytes, workspace_bytes);
        o.out = reinterpret_cast<float*>(workspace);
    }
    cudaStream_t st = as_stream(stream);
    const MfvConvA fa{mfv_geom(b, r, k), x, ldx, c, (int)K};
    const MatIn fb{dy, c_out};
    const dim3 grid((unsigned)((c_out + kMfvBN - 1) / kMfvBN), (unsigned)((K + kMfvBM - 1) / kMfvBM), (unsigned)pl.wsplits);
    train_gemm_kernel<kMfvBM, kMfvBN, false, true><<<grid, kGemmThreads, 0, st>>>(fa, fb, o, K, c_out, rows, pl.wkps);
    rc = check_launch("train_gemm_kernel");
    if (rc != PSA_OK || pl.wsplits == 1) return rc;
    return reduce_partials(pl.wsplits, (int)(K * c_out), o.out, dW, st);
}

extern "C" int psa_conv3d_bwd_data(int b, int r, int k, int c, int c_out, const float* dy, const float* W, float* dx, long long ld_dx,
                                   int accumulate, void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    int rc = mfv_bwd_dims("conv3d_bwd_data", b, r, k, c, c_out);
    if (rc != PSA_OK) return rc;
    PSA_REQUIRE(ld_dx >= c, "conv3d_bwd_data: row stride ld_dx=%lld below the width %d", ld_dx, c);
    if (b == 0) return PSA_OK;
    PSA_REQUIRE(dy && W && dx, "conv3d_bwd_data: null buffer");
    const MfvBwdPlan pl = mfv_bwd_plan(b, r, k, c, c_out);
    PSA_REQUIRE(workspace != nullptr && workspace_bytes >= pl.bytes,
                "conv3d_bwd_data: workspace of %zu bytes required (psa_conv3d_bwd_workspace_bytes), got %zu", pl.bytes, workspace_bytes);
    const long long rows = (long long)b * r * r * r;
    const int taps = k * k * k;
    GemmOut o;
    o.out = reinterpret_cast<float*>(workspace); o.ld_out = c; o.bias = nullptr; o.col_skip = 0; o.stat_partial = nullptr;
    cudaStream_t st = as_stream(stream);
    const MfvGradA fa{mfv_geom(b, r, k), dy, c_out, taps};
    const MfvWt fb{W, c, c_out};
    const dim3 grid((unsigned)((c + kMfvBN - 1) / kMfvBN), (unsigned)((rows + kMfvBM - 1) / kMfvBM), (unsigned)pl.dsplits);
    train_gemm_kernel<kMfvBM, kMfvBN, true, false><<<grid, kGemmThreads, 0, st>>>(fa, fb, o, rows, c, (long long)taps * c_out, pl.dkps);
    rc = check_launch("train_gemm_kernel");
    if (rc != PSA_OK) return rc;
    mfv_grad_finish_kernel<<<grid_for(rows * c), 256, 0, st>>>(pl.dsplits, rows, c, o.out, dx, ld_dx, accumulate ? 1 : 0);
    return check_launch("mfv_grad_finish_kernel");
}

extern "C" int psa_conv3d_bwd_macs(int b, int r, int k, int c, int c_out, long long* issued_weight, long long* issued_data,
                                   long long* in_grid) {
    int rc = mfv_bwd_dims("conv3d_bwd_macs", b, r, k, c, c_out);
    if (rc != PSA_OK) return rc;
    const MfvBwdPlan pl = mfv_bwd_plan(b < 1 ? 1 : b, r, k, c, c_out);
    const long long rows = (long long)b * r * r * r, K = (long long)k * k * k * c;
    const int taps = k * k * k;
    const MfvConvGeom g = mfv_geom(b, r, k);
    long long iw = 0, id = 0, ig = 0;
    for (int t = 0; t < taps && b > 0; ++t) {              // in grid: b * prod over the axes of (r - |offset|)
        int o[3];
        g.offset(t, o[0], o[1], o[2]);
        long long n = b;
        for (int a = 0; a < 3; ++a) n *= (r - (o[a] < 0 ? -o[a] : o[a])) > 0 ? r - (o[a] < 0 ? -o[a] : o[a]) : 0;
        ig += n * c * c_out;
    }
    if (b > 0) {
        const MfvConvA wa{g, nullptr, 0, c, (int)K};        // the kernels' own skip rule, tile by tile
        for (long long m0 = 0; m0 < K; m0 += kMfvBM)
            for (int sp = 0; sp < pl.wsplits; ++sp) {
                const long long kb = sp * pl.wkps, ke = kb + pl.wkps < rows ? kb + pl.wkps : rows;
                for (long long k0 = kb < ke ? wa.next_k(kb, ke, m0, kMfvBM) : ke; k0 < ke;) {
                    const long long kn = k0 + kGemmBK < ke ? wa.next_k(k0 + kGemmBK, ke, m0, kMfvBM) : ke;
                    iw += (k0 + kGemmBK < ke ? kGemmBK : ke - k0) * (m0 + kMfvBM < K ? kMfvBM : K - m0) * c_out;
                    k0 = kn;
                }
            }
        const MfvGradA da{g, nullptr, c_out, taps};
        const long long Kd = (long long)taps * c_out;
        for (long long m0 = 0; m0 < rows; m0 += kMfvBM)
            for (int sp = 0; sp < pl.dsplits; ++sp) {
                const long long kb = sp * pl.dkps, ke = kb + pl.dkps < Kd ? kb + pl.dkps : Kd;
                for (long long k0 = kb < ke ? da.next_k(kb, ke, m0, kMfvBM) : ke; k0 < ke;) {
                    const long long kn = k0 + kGemmBK < ke ? da.next_k(k0 + kGemmBK, ke, m0, kMfvBM) : ke;
                    id += (k0 + kGemmBK < ke ? kGemmBK : ke - k0) * (m0 + kMfvBM < rows ? kMfvBM : rows - m0) * c;
                    k0 = kn;
                }
            }
    }
    if (issued_weight) *issued_weight = iw;
    if (issued_data) *issued_data = id;
    if (in_grid) *in_grid = ig;
    return PSA_OK;
}

extern "C" int psa_mfv_bn_relu(long long rows, int C, const float* y, const float* scale, const float* shift, float* out, long long ldo,
                               psa_stream_t stream) {
    PSA_REQUIRE(rows >= 0 && C >= 1 && ldo >= C, "mfv_bn_relu: bad dims rows=%lld C=%d ldo=%lld", rows, C, ldo);
    if (rows == 0) return PSA_OK;
    PSA_REQUIRE(y && scale && shift && out, "mfv_bn_relu: null buffer");
    mfv_bn_relu_kernel<<<grid_for(rows * C), 256, 0, as_stream(stream)>>>(rows, C, y, scale, shift, out, ldo);
    return check_launch("mfv_bn_relu_kernel");
}

extern "C" int psa_mfv_bn_dy(long long rows, int C, const psa_grad_in* g, float* dy, psa_stream_t stream) {
    PSA_REQUIRE(rows >= 0 && C >= 1, "mfv_bn_dy: bad dims rows=%lld C=%d", rows, C);
    PSA_REQUIRE(g != nullptr && g->mode == 0, "mfv_bn_dy: a mode-0 psa_grad_in is required");
    if (rows == 0) return PSA_OK;
    PSA_REQUIRE(g->dh && dy && ((g->s == nullptr && g->ca == nullptr) || g->y), "mfv_bn_dy: null buffer");
    mfv_bn_dy_kernel<<<grid_for(rows * C), 256, 0, as_stream(stream)>>>(rows, C, GradIn(*g), dy);
    return check_launch("mfv_bn_dy_kernel");
}

extern "C" int psa_pool3d_max_train(int b, int r, int c, const float* x, float* out, unsigned char* winner, psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && r >= 1 && r < 256 && c >= 1, "pool3d_max_train: bad dims b=%d r=%d c=%d", b, r, c);
    if (b == 0) return PSA_OK;
    PSA_REQUIRE(x && out && winner, "pool3d_max_train: null buffer");
    const int ro = (r + 1) / 2;
    mfv_maxpool_win_kernel<<<grid_for((long long)b * ro * ro * ro * c), 256, 0, as_stream(stream)>>>(b, r, c, x, out, winner);
    return check_launch("mfv_maxpool_win_kernel");
}

extern "C" int psa_pool3d_bwd(int b, int r, int c, int kind, const float* dout, const unsigned char* winner, float* dx,
                              psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && r >= 1 && r < 256 && c >= 1, "pool3d_bwd: bad dims b=%d r=%d c=%d", b, r, c);
    PSA_REQUIRE(kind == 0 || kind == 1, "pool3d_bwd: kind=%d must be 0 (3^3 average) or 1 (2^3 max)", kind);
    if (b == 0) return PSA_OK;
    PSA_REQUIRE(dout && dx && (kind == 0 || winner), "pool3d_bwd: null buffer");
    const unsigned grid = grid_for((long long)b * r * r * r * c);
    if (kind == 0) {
        mfv_avgpool_bwd_kernel<<<grid, 256, 0, as_stream(stream)>>>(b, r, c, dout, dx);
        return check_launch("mfv_avgpool_bwd_kernel");
    }
    mfv_maxpool_bwd_kernel<<<grid, 256, 0, as_stream(stream)>>>(b, r, c, dout, winner, dx);
    return check_launch("mfv_maxpool_bwd_kernel");
}
