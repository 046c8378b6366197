/*
 * psa_oracle.c -- CPU restatement of the reference's point-set-abstraction arithmetic.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under scanobjectnn_b200/ may import, link or call this
 * file; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg
 * use it, and only as the checker or the CPU arm -- never as the product path.
 *
 * Every function cites the reference file:line it restates (paths relative to the reference
 * checkout, hkust-vgd/scanobjectnn @ 533e7e3).  Build: `make -C oracle` (gcc, -ffp-contract=off
 * so the ONLY fused multiply-adds are the fmaf() calls written below).
 *
 * Floating-point contract (verified from `cuobjdump -sass` of the reference .cu files compiled by
 * nvcc 12.9; the same contraction for sm_90a, see DESIGN.md "Arithmetic pinned from SASS"):
 *   GPU ops (FPS, ball query):  d2 = fma(dz,dz, fma(dx,dx, dy*dy))   -- FMUL(dy), FFMA(dx), FFMA(dz)
 *   CPU ops (three_nn, the test/ harness ball query): plain x86-64 g++ -O2, no FMA contraction:
 *                               d2 = (dx*dx + dy*dy) + dz*dz, each op rounded to float.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))

/* squared distance as the reference's CUDA kernels evaluate it after nvcc's contraction */
static inline float d2_gpu(float x1, float y1, float z1, float x2, float y2, float z2) {
    float dx = x2 - x1, dy = y2 - y1, dz = z2 - z1;
    float t = dy * dy;
    t = fmaf(dx, dx, t);
    t = fmaf(dz, dz, t);
    return t;
}
/* squared distance as a plain x86-64 (no FMA) build of the reference's CPU code evaluates it */
static inline float d2_cpu(float x1, float y1, float z1, float x2, float y2, float z2) {
    float dx = x2 - x1, dy = y2 - y1, dz = z2 - z1;
    float a = dx * dx;
    float b = dy * dy;
    float c = dz * dz;
    float s = a + b;
    return s + c;
}

/* ------------------------------------------------------------------------------------------------
 * Farthest point sampling.  Restates farthestpointsamplingKernel,
 * pointnet2/tf_ops/sampling/tf_sampling_g.cu:105-170 (launch <<<32,512>>>, :203-205):
 *   - seed index 0 (:114-116); running min-distance `temp` starts at 1e38 (:117-119)
 *   - thread t scans k = t, t+512, ... with strict `>` against best=-1 (:124-149)
 *   - min(d,td) is CUDA's fminf: a NaN distance leaves td unchanged (:143)
 *   - 9-level smem tree, `dists[i1]<dists[i2]` keeps the LOWER slot on ties (:152-162)
 * => winner among equal maxima is lexicographic in (k mod 512, k).
 * ------------------------------------------------------------------------------------------------ */
ORC_API void orc_fps(int b, int n, int m, const float* xyz, int* out) {
    if (m <= 0) return;
    enum { BS = 512 };
#pragma omp parallel for schedule(dynamic, 1)
    for (int i = 0; i < b; ++i) {
        const float* p = xyz + (size_t)i * n * 3;
        float* temp = (float*)malloc(sizeof(float) * (size_t)(n > 0 ? n : 1));
        float dists[BS];
        int dists_i[BS];
        for (int k = 0; k < n; ++k) temp[k] = 1e38f;
        int old = 0;
        out[(size_t)i * m] = old;
        for (int j = 1; j < m; ++j) {
            float x1 = p[old * 3 + 0], y1 = p[old * 3 + 1], z1 = p[old * 3 + 2];
            for (int t = 0; t < BS; ++t) {
                float best = -1.0f;
                int besti = 0;
                for (int k = t; k < n; k += BS) {
                    float td = temp[k];
                    float d = d2_gpu(x1, y1, z1, p[k * 3 + 0], p[k * 3 + 1], p[k * 3 + 2]);
                    float d2v = fminf(d, td);
                    if (d2v != td) temp[k] = d2v;
                    if (d2v > best) { best = d2v; besti = k; }
                }
                dists[t] = best;
                dists_i[t] = besti;
            }
            for (int u = 0; (1 << u) < BS; ++u) {
                for (int t = 0; t < (BS >> (u + 1)); ++t) {
                    int i1 = (t * 2) << u, i2 = (t * 2 + 1) << u;
                    if (dists[i1] < dists[i2]) { dists[i1] = dists[i2]; dists_i[i1] = dists_i[i2]; }
                }
            }
            old = dists_i[0];
            out[(size_t)i * m + j] = old;
        }
        free(temp);
    }
}

/* gatherpointKernel, tf_sampling_g.cu:172-181 */
ORC_API void orc_gather_point(int b, int n, int m, const float* inp, const int* idx, float* out) {
    for (int i = 0; i < b; ++i)
        for (int j = 0; j < m; ++j) {
            int a = idx[(size_t)i * m + j];
            for (int c = 0; c < 3; ++c) out[((size_t)i * m + j) * 3 + c] = inp[((size_t)i * n + a) * 3 + c];
        }
}

/* scatteraddpointKernel, tf_sampling_g.cu:183-192 (sequential order j = 0..m-1; the reference's
 * atomicAdd order is unspecified, so compare with a tolerance when indices repeat) */
ORC_API void orc_gather_point_grad(int b, int n, int m, const float* out_g, const int* idx, float* inp_g) {
    memset(inp_g, 0, sizeof(float) * (size_t)b * n * 3);
    for (int i = 0; i < b; ++i)
        for (int j = 0; j < m; ++j) {
            int a = idx[(size_t)i * m + j];
            for (int c = 0; c < 3; ++c) inp_g[((size_t)i * n + a) * 3 + c] += out_g[((size_t)i * m + j) * 3 + c];
        }
}

/* ------------------------------------------------------------------------------------------------
 * Ball query.  Restates query_ball_point_gpu, pointnet2/tf_ops/grouping/tf_grouping_g.cu:3-36
 * (identical control flow to test/query_ball_point.cpp:19-47): scan k in index order, keep the first
 * nsample with max(sqrtf(d2),1e-20f) < radius, on the first hit fill ALL slots with it, write pts_cnt.
 * `contract`=1 -> d2 as the CUDA op evaluates it; 0 -> as the x86 harness evaluates it.
 * `max` is fmaxf: a NaN distance becomes 1e-20 and therefore counts as inside (radius > 1e-20).
 * Queries with no hit leave their idx row untouched in the reference (uninitialised output,
 * tf_grouping.cpp:88); this restatement leaves the caller's buffer untouched too -- callers pre-fill.
 * ------------------------------------------------------------------------------------------------ */
ORC_API void orc_query_ball_point(int b, int n, int m, float radius, int nsample, const float* xyz1,
                                  const float* xyz2, int* idx, int* pts_cnt, int contract) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < b; ++i) {
        const float* p1 = xyz1 + (size_t)i * n * 3;
        const float* p2 = xyz2 + (size_t)i * m * 3;
        int* id = idx + (size_t)i * m * nsample;
        for (int j = 0; j < m; ++j) {
            int cnt = 0;
            float x2 = p2[j * 3 + 0], y2 = p2[j * 3 + 1], z2 = p2[j * 3 + 2];
            for (int k = 0; k < n; ++k) {
                if (cnt == nsample) break;
                float x1 = p1[k * 3 + 0], y1 = p1[k * 3 + 1], z1 = p1[k * 3 + 2];
                /* reference operand order: (x2-x1) with x2 the query (:20) */
                float dd = contract ? d2_gpu(x1, y1, z1, x2, y2, z2) : d2_cpu(x1, y1, z1, x2, y2, z2);
                float d = fmaxf(sqrtf(dd), 1e-20f);
                if (d < radius) {
                    if (cnt == 0)
                        for (int l = 0; l < nsample; ++l) id[j * nsample + l] = k;
                    id[j * nsample + cnt] = k;
                    cnt += 1;
                }
            }
            if (pts_cnt) pts_cnt[(size_t)i * m + j] = cnt;
        }
    }
}

/* group_point_gpu, tf_grouping_g.cu:40-57 */
ORC_API void orc_group_point(int b, int n, int c, int m, int nsample, const float* points, const int* idx,
                             float* out) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < b; ++i)
        for (int j = 0; j < m; ++j)
            for (int k = 0; k < nsample; ++k) {
                int ii = idx[((size_t)i * m + j) * nsample + k];
                memcpy(out + (((size_t)i * m + j) * nsample + k) * c, points + ((size_t)i * n + ii) * c,
                       sizeof(float) * (size_t)c);
            }
}

/* group_point_grad_gpu, tf_grouping_g.cu:61-78 (sequential summation order) */
ORC_API void orc_group_point_grad(int b, int n, int c, int m, int nsample, const float* grad_out,
                                  const int* idx, float* grad_points) {
    memset(grad_points, 0, sizeof(float) * (size_t)b * n * c);
    for (int i = 0; i < b; ++i)
        for (int j = 0; j < m; ++j)
            for (int k = 0; k < nsample; ++k) {
                int ii = idx[((size_t)i * m + j) * nsample + k];
                for (int l = 0; l < c; ++l)
                    grad_points[((size_t)i * n + ii) * c + l] += grad_out[(((size_t)i * m + j) * nsample + k) * c + l];
            }
}

/* ------------------------------------------------------------------------------------------------
 * SelectionSort.  Restates selection_sort_gpu, tf_grouping_g.cu:83-123: copy dist -> out, outi = s,
 * then k rounds of "find first strict minimum in [s+1,n), swap with slot s" carrying indices.
 * Ties are resolved by CURRENT ARRAY POSITION (after earlier swaps), not by original index.
 * ------------------------------------------------------------------------------------------------ */
ORC_API void orc_selection_sort(int b, int n, int m, int k, const float* dist, int* outi, float* out) {
#pragma omp parallel for schedule(static)
    for (int r = 0; r < b * m; ++r) {
        const float* d = dist + (size_t)r * n;
        float* o = out + (size_t)r * n;
        int* oi = outi + (size_t)r * n;
        for (int s = 0; s < n; ++s) { o[s] = d[s]; oi[s] = s; }
        for (int s = 0; s < k && s < n; ++s) {
            int mn = s;
            for (int t = s + 1; t < n; ++t)
                if (o[t] < o[mn]) mn = t;
            if (mn != s) {
                float tv = o[mn]; o[mn] = o[s]; o[s] = tv;
                int ti = oi[mn]; oi[mn] = oi[s]; oi[s] = ti;
            }
        }
    }
}

/* knn_point's distance matrix, tf_grouping.py:59-67: dist[b,j,i] = sum_c (xyz1[b,i,c]-xyz2[b,j,c])^2,
 * tf.reduce_sum over the last axis (c = 0..C-1, sequential, un-contracted: TF1 evaluates the
 * subtract / square / reduce_sum as separate ops, so no FMA can form across them). */
ORC_API void orc_knn_point_dist(int b, int n, int m, int c, const float* xyz1, const float* xyz2, float* dist) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < b; ++i)
        for (int j = 0; j < m; ++j)
            for (int k = 0; k < n; ++k) {
                float s = 0.0f;
                for (int l = 0; l < c; ++l) {
                    float df = xyz1[((size_t)i * n + k) * c + l] - xyz2[((size_t)i * m + j) * c + l];
                    float sq = df * df;
                    s = s + sq;
                }
                dist[((size_t)i * m + j) * n + k] = s;
            }
}

/* ------------------------------------------------------------------------------------------------
 * three_nn.  Restates threenn_cpu, pointnet2/tf_ops/3d_interpolation/tf_interpolate.cpp:60-103:
 * distance expression evaluated in float (x86, un-contracted) then widened to double; best1..3 start
 * at 1e40 (-> +inf when stored to float); strict `<` cascade, so the earlier k wins ties.
 * ------------------------------------------------------------------------------------------------ */
ORC_API void orc_three_nn(int b, int n, int m, const float* xyz1, const float* xyz2, float* dist, int* idx) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < b; ++i) {
        const float* p1 = xyz1 + (size_t)i * n * 3;
        const float* p2 = xyz2 + (size_t)i * m * 3;
        for (int j = 0; j < n; ++j) {
            float x1 = p1[j * 3 + 0], y1 = p1[j * 3 + 1], z1 = p1[j * 3 + 2];
            double best1 = 1e40, best2 = 1e40, best3 = 1e40;
            int bi1 = 0, bi2 = 0, bi3 = 0;
            for (int k = 0; k < m; ++k) {
                double d = (double)d2_cpu(x1, y1, z1, p2[k * 3 + 0], p2[k * 3 + 1], p2[k * 3 + 2]);
                if (d < best1) { best3 = best2; bi3 = bi2; best2 = best1; bi2 = bi1; best1 = d; bi1 = k; }
                else if (d < best2) { best3 = best2; bi3 = bi2; best2 = d; bi2 = k; }
                else if (d < best3) { best3 = d; bi3 = k; }
            }
            size_t o = ((size_t)i * n + j) * 3;
            dist[o + 0] = (float)best1; idx[o + 0] = bi1;
            dist[o + 1] = (float)best2; idx[o + 1] = bi2;
            dist[o + 2] = (float)best3; idx[o + 2] = bi3;
        }
    }
}

/* threeinterpolate_cpu, tf_interpolate.cpp:107-127: out = p[i1]*w1 + p[i2]*w2 + p[i3]*w3,
 * evaluated left to right in float, un-contracted (x86-64 baseline build). */
ORC_API void orc_three_interpolate(int b, int m, int c, int n, const float* points, const int* idx,
                                   const float* weight, float* out) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < b; ++i)
        for (int j = 0; j < n; ++j) {
            size_t o = ((size_t)i * n + j) * 3;
            float w1 = weight[o], w2 = weight[o + 1], w3 = weight[o + 2];
            const float* q1 = points + ((size_t)i * m + idx[o]) * c;
            const float* q2 = points + ((size_t)i * m + idx[o + 1]) * c;
            const float* q3 = points + ((size_t)i * m + idx[o + 2]) * c;
            for (int l = 0; l < c; ++l) {
                float a = q1[l] * w1;
                float bb = q2[l] * w2;
                float cc = q3[l] * w3;
                float s = a + bb;
                out[((size_t)i * n + j) * c + l] = s + cc;
            }
        }
}

/* threeinterpolate_grad_cpu, tf_interpolate.cpp:131-153 (sequential accumulation order) */
ORC_API void orc_three_interpolate_grad(int b, int n, int c, int m, const float* grad_out, const int* idx,
                                        const float* weight, float* grad_points) {
    memset(grad_points, 0, sizeof(float) * (size_t)b * m * c);
    for (int i = 0; i < b; ++i)
        for (int j = 0; j < n; ++j) {
            size_t o = ((size_t)i * n + j) * 3;
            for (int t = 0; t < 3; ++t) {
                float w = weight[o + t];
                float* g = grad_points + ((size_t)i * m + idx[o + t]) * c;
                for (int l = 0; l < c; ++l) g[l] += grad_out[((size_t)i * n + j) * c + l] * w;
            }
        }
}

/* pointnet_fp_module's weights, pointnet2/utils/pointnet_util.py:212-215:
 * dist=max(dist,1e-10); norm=sum(1/dist); weight=(1/dist)/norm  (tf.reduce_sum over 3, in order) */
ORC_API void orc_three_weights(int rows, const float* dist, float* weight) {
    for (int r = 0; r < rows; ++r) {
        float r0 = 1.0f / fmaxf(dist[r * 3 + 0], 1e-10f);
        float r1 = 1.0f / fmaxf(dist[r * 3 + 1], 1e-10f);
        float r2 = 1.0f / fmaxf(dist[r * 3 + 2], 1e-10f);
        float s = r0 + r1;
        s = s + r2;
        weight[r * 3 + 0] = r0 / s;
        weight[r * 3 + 1] = r1 / s;
        weight[r * 3 + 2] = r2 / s;
    }
}

/* ------------------------------------------------------------------------------------------------
 * DGCNN kNN graph.  Restates dgcnn/utils/tf_util.py:638-671:
 *   inner = -2 * (X . X^T)                      (tf.matmul, :653-654)
 *   sq    = sum_c x_c^2                         (:655)
 *   adj   = sq_i + inner_ij + sq_j              (:657, left to right)
 *   nn    = top_k(-adj, k)                      (:670) -> ascending adj, lower index first on ties
 * The matmul / reduce_sum accumulation order inside TensorFlow/cuBLAS is NOT pinned by the
 * reference (parity unpinned, SURVEY 8c).  Declared canonical order, shared with the CUDA kernel:
 *   dot = fma chain over c = 0..C-1 starting from 0.0f (dot = fmaf(x_ic, x_jc, dot));
 *   sq  = fma chain over c = 0..C-1 starting from 0.0f;
 *   adj = (sq_i + (-2.0f*dot)) + sq_j.
 * `adj_out` (b,n,n) optional.
 * ------------------------------------------------------------------------------------------------ */
ORC_API void orc_dgcnn_knn(int b, int n, int c, int k, const float* x, float* adj_out, int* nn_idx) {
#pragma omp parallel for schedule(dynamic, 1)
    for (int i = 0; i < b; ++i) {
        const float* X = x + (size_t)i * n * c;
        float* sq = (float*)malloc(sizeof(float) * (size_t)n);
        float* row = (float*)malloc(sizeof(float) * (size_t)n);
        unsigned char* taken = (unsigned char*)malloc((size_t)n);
        for (int p = 0; p < n; ++p) {
            float s = 0.0f;
            for (int l = 0; l < c; ++l) s = fmaf(X[(size_t)p * c + l], X[(size_t)p * c + l], s);
            sq[p] = s;
        }
        for (int p = 0; p < n; ++p) {
            for (int q = 0; q < n; ++q) {
                float dot = 0.0f;
                for (int l = 0; l < c; ++l) dot = fmaf(X[(size_t)p * c + l], X[(size_t)q * c + l], dot);
                float inner = -2.0f * dot;
                float a = sq[p] + inner;
                row[q] = a + sq[q];
            }
            if (adj_out) memcpy(adj_out + ((size_t)i * n + p) * n, row, sizeof(float) * (size_t)n);
            if (nn_idx) {
                memset(taken, 0, (size_t)n);
                for (int s = 0; s < k; ++s) {
                    int best = -1;
                    for (int q = 0; q < n; ++q)
                        if (!taken[q] && (best < 0 || row[q] < row[best])) best = q;
                    taken[best] = 1;
                    nn_idx[((size_t)i * n + p) * k + s] = best;
                }
            }
        }
        free(sq); free(row); free(taken);
    }
}

/* top_k(-adj,k) on a caller-provided matrix (dgcnn/utils/tf_util.py:660-671) */
ORC_API void orc_topk_smallest(int rows, int n, int k, const float* adj, int* nn_idx) {
#pragma omp parallel for schedule(static)
    for (int r = 0; r < rows; ++r) {
        const float* row = adj + (size_t)r * n;
        unsigned char* taken = (unsigned char*)calloc((size_t)n, 1);
        for (int s = 0; s < k; ++s) {
            int best = -1;
            for (int q = 0; q < n; ++q)
                if (!taken[q] && (best < 0 || row[q] < row[best])) best = q;
            taken[best] = 1;
            nn_idx[(size_t)r * k + s] = best;
        }
        free(taken);
    }
}
