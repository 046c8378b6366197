/*
 * pointcnn_knn.c -- CPU restatement of PointCNN's dilated kNN, the checker of psa_knn_dilated.
 *
 * TEST INFRASTRUCTURE ONLY.  oracle/pointcnn_oracle.py compiles this file on first use (gcc, -ffp-contract=off, so the ONLY
 * fused multiply-adds are the fmaf() calls written below); nothing under scanobjectnn_b200/ may import, link or call it.
 *
 * Restates PointCNN/pointfly.py:163-176 knn_indices_general(queries, points, k*d, sort=True) and pointcnn.py:12-13
 * (indices_dilated[:, :, ::d]):
 *   D    = r_q - 2 (q . p) + r_p                  (batch_distance_matrix_general, pointfly.py:122-128)
 *   nn   = top_k(-D, k*d)                         -> ascending D, lower index first on ties
 *   keep every d-th entry, starting with the first.
 * unique=True changes nothing: prepare_for_unique_top_k adds to its local name (pointfly.py:142-144).
 * The reference's matmul / reduce_sum order is not pinned; the canonical fp32 order is the one oracle/psa_oracle.c:orc_dgcnn_knn
 * declares for DGCNN, here for 3 channels: dot and the squared norms are fma chains over x, y, z from 0.0f, and
 * D = (sq_q + (-2.0f*dot)) + sq_p.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))

/* points (b,n,3), queries (b,m,3) -> nn_idx (b,m,k); k*d <= n */
ORC_API void orc_knn_dilated(int b, int n, int m, int k, int d, const float* points, const float* queries, int* nn_idx) {
    const int L = k * d;
#pragma omp parallel for schedule(dynamic, 1)
    for (int i = 0; i < b; ++i) {
        const float* X = points + (size_t)i * n * 3;
        const float* Q = queries + (size_t)i * m * 3;
        float* sq = (float*)malloc(sizeof(float) * (size_t)n);
        float* row = (float*)malloc(sizeof(float) * (size_t)n);
        unsigned char* taken = (unsigned char*)malloc((size_t)n);
        for (int p = 0; p < n; ++p) {
            float s = 0.0f;
            for (int l = 0; l < 3; ++l) s = fmaf(X[(size_t)p * 3 + l], X[(size_t)p * 3 + l], s);
            sq[p] = s;
        }
        for (int qi = 0; qi < m; ++qi) {
            const float* q = Q + (size_t)qi * 3;
            float sq_q = 0.0f;
            for (int l = 0; l < 3; ++l) sq_q = fmaf(q[l], q[l], sq_q);
            for (int p = 0; p < n; ++p) {
                float dot = 0.0f;
                for (int l = 0; l < 3; ++l) dot = fmaf(q[l], X[(size_t)p * 3 + l], dot);
                float inner = -2.0f * dot;
                float a = sq_q + inner;
                row[p] = a + sq[p];
            }
            memset(taken, 0, (size_t)n);
            for (int s = 0; s < L; ++s) {
                int best = -1;
                for (int p = 0; p < n; ++p)
                    if (!taken[p] && (best < 0 || row[p] < row[best])) best = p;
                taken[best] = 1;
                if (s % d == 0) nn_idx[((size_t)i * m + qi) * k + s / d] = best;
            }
        }
        free(sq); free(row); free(taken);
    }
}
