/*
 * psa.h -- C ABI of libpsa.so: the H100-native (sm_90a) point-set-abstraction hot path.
 *
 * This is the drop-in boundary.  The reference (hkust-vgd/scanobjectnn) reaches its native code through
 * plain C++ "Launcher" functions called from TensorFlow OpKernel::Compute (raw device pointers + int
 * dims, caller-owned buffers); every entry point below names the reference interface it replaces.
 * Reference paths are relative to pointnet2/tf_ops/ unless they start with dgcnn/ or pointnet2/.
 *
 * Conventions (all entry points):
 *   - every pointer is a DEVICE pointer to a dense, contiguous, row-major fp32 / int32 buffer owned by
 *     the caller; nothing is allocated or freed inside the library; outputs must not alias inputs;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream, which is what the
 *     reference's `<<<grid,block>>>` launches use); calls are asynchronous on that stream;
 *   - return value: PSA_OK (0); PSA_ERR_INVALID_ARGUMENT (-1) for a shape/attribute the reference's
 *     OP_REQUIRES would reject (message via psa_last_error()); PSA_ERR_UNSUPPORTED (-2) for a shape
 *     outside the compiled limits; a positive value is the cudaError_t of a failed launch.  Unlike the
 *     reference (which never checks), launches are checked with cudaGetLastError();
 *   - b == 0 or an empty extent is a successful no-op;
 *   - thread-safe: no global mutable state except the thread-local error string.
 */
#ifndef PSA_H_
#define PSA_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PSA_OK 0
#define PSA_ERR_INVALID_ARGUMENT (-1)
#define PSA_ERR_UNSUPPORTED (-2)

typedef void* psa_stream_t; /* cudaStream_t */

#if defined(__GNUC__)
#define PSA_API __attribute__((visibility("default")))
#else
#define PSA_API
#endif

/* library identity / diagnostics */
PSA_API int psa_version(void);                 /* MAJOR*10000 + MINOR*100 + PATCH */
PSA_API const char* psa_last_error(void);      /* thread-local, valid until the next failing call on this thread */
PSA_API int psa_sm_arch(void);                 /* 90: the only architecture compiled in (sm_90a) */

/* ---------------------------------------------------------------------------------------------
 * sampling/  (tf_sampling.cpp, tf_sampling_g.cu)
 * ------------------------------------------------------------------------------------------- */

/* Farthest point sampling.  Replaces
 *   void farthestpointsamplingLauncher(int b,int n,int m,const float* inp,float* temp,int* out)
 *   (sampling/tf_sampling.cpp:94, kernel tf_sampling_g.cu:105-170; op FarthestPointSample :28-40).
 * xyz (b,n,3) -> idx (b,m) int32; seed index 0; ties between equal maxima resolved exactly as the
 * reference's 512-thread strided scan + tree do: minimum over (k mod 512, k).  No `temp` scratch is
 * needed (running distances live in registers).  If new_xyz != NULL the gather of the sampled points
 * (GatherPoint, below) is fused: new_xyz (b,m,3).  Requires n >= 1 when m >= 1; m may exceed n. */
PSA_API int psa_farthest_point_sample(int b, int n, int m, const float* xyz, int* idx, float* new_xyz,
                              psa_stream_t stream);

/* Replaces gatherpointLauncher (sampling/tf_sampling.cpp:125, tf_sampling_g.cu:172-181).
 * inp (b,n,3), idx (b,m) -> out (b,m,3). */
PSA_API int psa_gather_point(int b, int n, int m, const float* inp, const int* idx, float* out, psa_stream_t stream);

/* Replaces cudaMemset + scatteraddpointLauncher (sampling/tf_sampling.cpp:150,174; tf_sampling_g.cu:183-192).
 * out_g (b,m,3), idx (b,m) -> inp_g (b,n,3), every element written.  Ordered (no float atomics): see
 * psa_scatter_workspace_bytes(b, n, m). */
PSA_API int psa_gather_point_grad(int b, int n, int m, const float* out_g, const int* idx, float* inp_g, void* workspace,
                          size_t workspace_bytes, psa_stream_t stream);

/* The three scatter-add gradients (GatherPointGrad, GroupPointGrad, ThreeInterpolateGrad) add the contributions of one
 * destination in ascending entry order -- the order of the reference's sequential CPU loops (grouping/test/ ..._cpu, tf_interpolate.cpp)
 * -- instead of the float atomicAdd of its CUDA kernels: results are bit-reproducible.  They need a device scratch buffer of
 * this many bytes for the per-cloud (destination -> entries) lists: b clouds, n_dst destination points and `entries`
 * scattered rows per cloud (m; m*nsample; 3*n).  Out-of-range indices are dropped.  n_dst <= 51200. */
PSA_API size_t psa_scatter_workspace_bytes(int b, int n_dst, long long entries);

/* ---------------------------------------------------------------------------------------------
 * grouping/  (tf_grouping.cpp, tf_grouping_g.cu)
 * ------------------------------------------------------------------------------------------- */

/* Replaces queryBallPointLauncher (grouping/tf_grouping.cpp:66, tf_grouping_g.cu:3-36; op QueryBallPoint :13-30).
 * xyz1 (b,n,3) dataset, xyz2 (b,m,3) queries -> idx (b,m,nsample), pts_cnt (b,m).
 * First `nsample` points in index order with max(sqrtf(d2),1e-20f) < radius; unused slots repeat the
 * first hit.  A query with an empty ball gets idx row = 0 and pts_cnt = 0 (the reference leaves that
 * row uninitialised).  pts_cnt may be NULL. */
PSA_API int psa_query_ball_point(int b, int n, int m, float radius, int nsample, const float* xyz1, const float* xyz2,
                         int* idx, int* pts_cnt, psa_stream_t stream);

/* Replaces groupPointLauncher (grouping/tf_grouping.cpp:142, tf_grouping_g.cu:40-57).
 * points (b,n,c), idx (b,m,nsample) -> out (b,m,nsample,c). */
PSA_API int psa_group_point(int b, int n, int c, int m, int nsample, const float* points, const int* idx, float* out,
                    psa_stream_t stream);

/* Replaces cudaMemset + groupPointGradLauncher (grouping/tf_grouping.cpp:173,204; tf_grouping_g.cu:61-78).
 * grad_out (b,m,nsample,c), idx -> grad_points (b,n,c), every element written.
 * workspace: psa_scatter_workspace_bytes(b, n, m*nsample). */
PSA_API int psa_group_point_grad(int b, int n, int c, int m, int nsample, const float* grad_out, const int* idx,
                         float* grad_points, void* workspace, size_t workspace_bytes, psa_stream_t stream);

/* Replaces selectionSortLauncher (grouping/tf_grouping.cpp:108, tf_grouping_g.cu:83-123; op SelectionSort).
 * dist (b,m,n) -> outi (b,m,n) int32, out (b,m,n): full copies whose first k slots per row hold the k
 * smallest, produced by the reference's swap-based partial selection sort (ties by current position). */
PSA_API int psa_selection_sort(int b, int n, int m, int k, const float* dist, int* outi, float* out, psa_stream_t stream);

/* knn_point (grouping/tf_grouping.py:49-74) without the (b,m,n) matrices: xyz1 (b,n,c) dataset,
 * xyz2 (b,m,c) queries -> val (b,m,k), idx (b,m,k); same distances (sum_c (a-b)^2, sequential,
 * un-contracted) and the same swap-based tie order as SelectionSort. */
PSA_API int psa_knn_point(int b, int n, int m, int c, int k, const float* xyz1, const float* xyz2, float* val, int* idx,
                  psa_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * 3d_interpolation/  (tf_interpolate.cpp -- CPU-only ops in the reference)
 * ------------------------------------------------------------------------------------------- */

/* Replaces threenn_cpu (3d_interpolation/tf_interpolate.cpp:60-103; op ThreeNN :12-21).
 * xyz1 (b,n,3) unknown, xyz2 (b,m,3) known -> dist (b,n,3) SQUARED distances ascending, idx (b,n,3).
 * Strict-< cascade (earlier k wins ties); slots beyond m are dist=+inf, idx=0. */
PSA_API int psa_three_nn(int b, int n, int m, const float* xyz1, const float* xyz2, float* dist, int* idx,
                 psa_stream_t stream);

/* Replaces threeinterpolate_cpu (tf_interpolate.cpp:107-127).
 * points (b,m,c), idx (b,n,3), weight (b,n,3) -> out (b,n,c) = (p1*w1 + p2*w2) + p3*w3. */
PSA_API int psa_three_interpolate(int b, int m, int c, int n, const float* points, const int* idx, const float* weight,
                          float* out, psa_stream_t stream);

/* Replaces memset + threeinterpolate_grad_cpu (tf_interpolate.cpp:131-153,258).
 * grad_out (b,n,c), idx, weight -> grad_points (b,m,c), every element written; bit-identical to the reference's CPU loop
 * (same order, product rounded before the add).  workspace: psa_scatter_workspace_bytes(b, m, 3*n). */
PSA_API int psa_three_interpolate_grad(int b, int n, int c, int m, const float* grad_out, const int* idx,
                               const float* weight, float* grad_points, void* workspace, size_t workspace_bytes,
                               psa_stream_t stream);

/* The interpolation half of pointnet_fp_module (pointnet2/utils/pointnet_util.py:211-216) in one launch:
 * three_nn -> dist=max(dist,1e-10) -> w=(1/dist)/sum(1/dist) -> three_interpolate.
 * Optional outputs dist/idx/weight (b,n,3) may be NULL. */
PSA_API int psa_three_nn_interpolate(int b, int n, int m, int c, const float* xyz1, const float* xyz2,
                             const float* points2, float* out, float* dist, int* idx, float* weight,
                             psa_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * input pipeline  (data_utils.py:133-186, pointnet2/utils/provider.py:34-52,189-236, train.py:246-252 -- numpy on the
 * host in the reference, one kernel here).  src (b,n_src,3) -> out (b,n,3):
 *   [center over all n_src points] -> [divide by the max norm] -> gather perm[0..n) (same subset for every cloud; NULL =
 *   the first n points) -> [dropout: dropped points := the cloud's first batch point] -> [rotate about the up axis by
 *   (cos,sin) given in double, float64 product] -> [scale (b)] -> [shift (b,3)] -> [+ clip(sigma * noise, -clip, clip),
 *   float64 sum].  Every optional input may be NULL (step skipped).  The random numbers are inputs; see ops.augment_batch.
 * ------------------------------------------------------------------------------------------- */
PSA_API int psa_augment_batch(int b, int n_src, int n, const float* src, const int* perm, const double* cos_sin,
                              const float* scale, const float* shift, const float* noise, double sigma, double clip,
                              const unsigned char* drop, int center, int normalize, float* out, psa_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * dgcnn graph functions  (dgcnn/utils/tf_util.py:638-706 -- TF library ops in the reference)
 * ------------------------------------------------------------------------------------------- */

/* pairwise_distance (dgcnn/utils/tf_util.py:638-657): x (b,n,c) -> adj (b,n,n),
 * adj = (|x_i|^2 + (-2 x_i.x_j)) + |x_j|^2 with fma chains over c (canonical order, oracle/psa_oracle.c). */
PSA_API int psa_pairwise_distance(int b, int n, int c, const float* x, float* adj, psa_stream_t stream);

/* knn (dgcnn/utils/tf_util.py:660-671): adj (b,n,ncols) -> nn_idx (b,n,k): top_k(-adj), ascending adj,
 * lower index first on ties. */
PSA_API int psa_knn_topk(int b, int n, int ncols, int k, const float* adj, int* nn_idx, psa_stream_t stream);

/* pairwise_distance + knn fused, never materialising (b,n,n): x (b,n,c) -> nn_idx (b,n,k). */
PSA_API int psa_knn_graph(int b, int n, int c, int k, const float* x, int* nn_idx, psa_stream_t stream);

/* get_edge_feature (dgcnn/utils/tf_util.py:674-706): x (b,n,c), nn_idx (b,n,k) -> (b,n,k,2c) = [x_i, x_j-x_i]. */
PSA_API int psa_get_edge_feature(int b, int n, int c, int k, const float* x, const int* nn_idx, float* out,
                         psa_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * grouped shared MLP  (pointnet2/utils/pointnet_util.py:87-154, tf_util.conv2d 1x1 + BN + ReLU,
 * dgcnn EdgeConv dgcnn/models/dgcnn.py:31-80) -- TF/cuDNN library ops in the reference
 * ------------------------------------------------------------------------------------------- */

/* One per-row shared MLP: up to PSA_MAX_MLP_LAYERS layers of  y = relu?( (x . W) * scale + shift ).
 *   channels[0..n_layers]   C_0 (input) ... C_L
 *   weight[l]  (C_l, C_{l+1}) row-major  == TF conv kernel (1,1,C_in,C_out) (tf_util.py:162-168)
 *   scale[l], shift[l]  (C_{l+1}): conv bias + inference-mode batch norm folded by the caller:
 *        scale = gamma / sqrt(moving_var + 1e-3),  shift = (bias - moving_mean) * scale + beta
 *        (no BN: scale = 1, shift = bias);  scale[l] may be NULL (= all ones)
 *   relu[l]    nonzero -> ReLU after layer l */
#define PSA_MAX_MLP_LAYERS 4
typedef struct psa_mlp {
    int n_layers;
    int channels[PSA_MAX_MLP_LAYERS + 1];
    const float* weight[PSA_MAX_MLP_LAYERS];
    const float* scale[PSA_MAX_MLP_LAYERS];
    const float* shift[PSA_MAX_MLP_LAYERS];
    int relu[PSA_MAX_MLP_LAYERS];
    /* Optional, for weights that do not change between calls (inference): tensor-core weight images built ONCE by
     * psa_prepare_weight_image().  image[l] == NULL -> the entry point builds the image in its workspace on every call
     * (~45 us per PointNet++ forward).  An image is only used if its tile width / first row match what the entry point
     * needs (psa_mlp_image_plan() tells); otherwise it is ignored and rebuilt. */
    const void* image[PSA_MAX_MLP_LAYERS];
    int image_nt[PSA_MAX_MLP_LAYERS];      /* tile width the image was built for, as returned by psa_mlp_image_plan (64 or 128, | 0x200 = fp16x2 blocks followed by their bf16x3 twin, | 0x100 = bf16x3 only) */
    int image_row0[PSA_MAX_MLP_LAYERS];    /* first row of weight[l] covered by the image (3 when the xyz rows are split off) */
} psa_mlp;

/* Which images would an entry point use for this MLP?  usage: 0 = psa_shared_mlp(rows, pool_k), 1 = psa_sa_group_all_infer
 * (rows = b*n, c), 2 = psa_sa_module_infer (rows = b*n, c, nsample).  Fills nt/row0/bytes per layer (bytes 0 = that layer
 * does not run on the tensor cores).  Returns PSA_OK. */
#define PSA_USAGE_SHARED_MLP 0
#define PSA_USAGE_SA_GROUP_ALL 1
#define PSA_USAGE_SA_MODULE 2
PSA_API int psa_mlp_image_plan(int usage, long long rows, int pool_k, int c, int nsample, const psa_mlp* mlp,
                               int nt[PSA_MAX_MLP_LAYERS], int row0[PSA_MAX_MLP_LAYERS], size_t bytes[PSA_MAX_MLP_LAYERS]);
/* Build the image of rows [row0, K) of W (K, N) for tile width | format `nt` into `image` (bytes from psa_mlp_image_plan).
 * An fp16x2 image is followed, in the same buffer, by the bf16x3 image the range guard reruns on. */
PSA_API int psa_prepare_weight_image(int K, int N, int row0, int nt, const float* W, void* image, psa_stream_t stream);

/* Dense rows: x (rows, C_0) -> out.  pool_k == 1: out (rows, C_L).  pool_k > 1: rows must be a multiple
 * of pool_k and out (rows/pool_k, C_L) = channel-wise max over each run of pool_k consecutive rows
 * (tf.reduce_max over nsample, pointnet_util.py:127); pool_k must divide 128 (>= 8) or be a multiple of 128.
 * Used for sample_and_group_all (SA3), FP-module convs, DGCNN's point-wise convs and the FC heads.
 * Layers run one launch each; the (rows, C_l) intermediates ping-pong through the caller's workspace of
 * psa_shared_mlp_workspace_bytes(rows, mlp) bytes (0 for a single layer; workspace may then be NULL). */
PSA_API size_t psa_shared_mlp_workspace_bytes(long long rows, const psa_mlp* mlp);
PSA_API int psa_shared_mlp(long long rows, int pool_k, const float* x, const psa_mlp* mlp, float* out,
                           void* workspace, size_t workspace_bytes, psa_stream_t stream);

/* psa_shared_mlp (pool_k = 1) whose first layer also takes one input row per group of group_rows consecutive rows:
 *   layer 0:  relu?( (x[r] . W0 + group_add[r / group_rows]) * scale0 + shift0 ),  group_add (rows / group_rows, C_1)
 * and the later layers as in psa_shared_mlp.  This is a 1x1 conv over concat([x, tile(g, group_rows)]) (pointnet/models/
 * pointnet_seg.py:81-88) without the concatenation: with W = [W_x ; W_g] (x rows first), group_add = g . W_g is one
 * psa_shared_mlp call over the groups, and the layer over the rows has K = C_0 = the width of x only.  group_rows must
 * divide rows (else PSA_ERR_INVALID_ARGUMENT); groups need not align with the kernels' row tiles.  Same workspace as
 * psa_shared_mlp (psa_shared_mlp_workspace_bytes). */
PSA_API int psa_shared_mlp_grouped(long long rows, long long group_rows, const float* x, const psa_mlp* mlp, const float* group_add,
                                   float* out, void* workspace, size_t workspace_bytes, psa_stream_t stream);

/* Fused set-abstraction level, inference mode (pointnet_sa_module, pointnet_util.py:87-154 with
 * sample_and_group :22-56 inside): for every query j of new_xyz
 *   idx_j  = query_ball_point(radius, nsample, xyz, new_xyz)[j]           (or caller-provided idx)
 *   row_k  = [ xyz[idx_jk] - new_xyz[j]  ,  points[idx_jk] ]               (xyz first, :46-50)
 *   out_j  = max_k  MLP(row_k)
 * without materialising the (b,m,nsample,3+c) tensor.  xyz (b,n,3), new_xyz (b,m,3), points (b,n,c) or
 * NULL with c = 0, mlp->channels[0] must equal 3 + c.  out (b,m,C_L).
 * idx_in  != NULL: use these neighbourhoods (b,m,nsample) instead of searching;
 * idx_out != NULL / pts_cnt != NULL: also write the ball-query result (idx_out is REQUIRED when idx_in is NULL).
 * workspace: psa_sa_module_workspace_bytes() bytes of device scratch (per-point layer-1 products), may be 0/NULL. */
PSA_API size_t psa_sa_module_workspace_bytes(int b, int n, int m, int c, int nsample, const psa_mlp* mlp);
PSA_API int psa_sa_module_infer(int b, int n, int m, int c, float radius, int nsample, const float* xyz,
                                const float* new_xyz, const float* points, const int* idx_in, const psa_mlp* mlp,
                                float* out, int* idx_out, int* pts_cnt, void* workspace, size_t workspace_bytes,
                                psa_stream_t stream);

/* pointnet_sa_module with group_all=True (pointnet_util.py:59-84,113-127): rows [xyz, points] (xyz first) -> MLP -> max over
 * the n points of each cloud, without building the (b,n,3+c) concatenation.  xyz (b,n,3), points (b,n,c), mlp->channels[0]
 * == 3 + c -> out (b, C_L).  Returns PSA_ERR_UNSUPPORTED when the first layer cannot run on the tensor-core path (then
 * concatenate and call psa_shared_mlp with pool_k = n). */
PSA_API size_t psa_sa_group_all_workspace_bytes(int b, int n, int c, const psa_mlp* mlp);
PSA_API int psa_sa_group_all_infer(int b, int n, int c, const float* xyz, const float* points, const psa_mlp* mlp,
                                   float* out, void* workspace, size_t workspace_bytes, psa_stream_t stream);

/* Arithmetic of the grouped MLP.  Whenever the shapes allow -- set-abstraction levels with widths 64/128 (last width 64 or a
 * multiple of 128) and nsample 32/64/128 on tc_sa_kernel, dense layers with N = 64 or a multiple of 128 on tc_dense_kernel
 * -- the layers after the first run on the Hopper tensor cores (wgmma) with fp32 accumulation; other shapes
 * run on the fp32-FMA kernels.  The fp32 operands are split into exactly representable 16-bit pieces:
 *   0 (default): two fp16 pieces per operand, three MMAs per product  a1w2 + a2w1 + a1w1.  Each output column of a weight image
 *      is scaled by a power of two 2^e_n that brings its largest |w| into [2^10, 2^11) before the split, and 2^-e_n is folded into
 *      the layer's scale (exact): every weight keeps 22 bits relative to the largest weight of its column, at any weight scale.
 *      Activations are split unscaled and keep an absolute 2^-25 (fp16's subnormal step), which is below the 1e-5 contract
 *      of the tests for the O(1) post-batch-norm activations and coordinates the models feed their layers; with batch norm
 *      calibrated to the data (folded scales up to 31.6 gamma) the layers stay within 1e-5 of fp64.  fp16 covers |v| < 65504:
 *      the kernels track the activation pieces they store and raise a device-side flag when one leaves that range or a weight
 *      is not finite; the call then reruns the op with bf16x3 operands (launched unconditionally, a no-op unless the flag is set),
 *      so results are valid for any fp32 input.
 *   2: three bf16 pieces per operand, six MMAs per product (small terms first) -- any magnitude, twice the tensor work.
 *   1: fp32-FMA kernels only.
 * Weight images (psa_prepare_weight_image) are format-specific: psa_mlp_image_plan returns the format of the current mode in its
 * nt values; images of the other format are ignored (rebuilt per call).  The switch is process-global (two atomics: changing it while
 * other threads launch is race-free, but a call in flight may see either mode for its later layers): set it before launching
 * work, not concurrently with it. */
PSA_API int psa_set_mlp_mode(int mode);
PSA_API int psa_get_mlp_mode(void);

/* Training-mode front of a set-abstraction level ("variant F1"): ball query + group + centre + first 1x1 conv + bias in
 * one launch, writing the PRE-batch-norm activations (which training-mode BN needs in HBM once: batch statistics come
 * before the ReLU, pointnet2/utils/tf_util.py:512-531 with is_training=True) and, optionally, their per-channel sum and
 * sum of squares.  xyz (b,n,3), new_xyz (b,m,3), points (b,n,c) or NULL, w1 (3+c, C1) (xyz rows first), bias (C1) or
 * NULL -> pre (b,m,nsample,C1), idx (b,m,nsample), pts_cnt (b,m) or NULL, stats (2,C1) or NULL.  C1 in {64,128}.
 * Replaces query_ball_point + group_point x2 + tile/sub + concat + conv2d/bias_add (pointnet_util.py:44-50,117-123). */
PSA_API size_t psa_sa_conv1_prebn_workspace_bytes(int b, int n, int m, int c, int C1, int want_stats);
PSA_API int psa_sa_conv1_prebn(int b, int n, int m, int c, float radius, int nsample, const float* xyz,
                               const float* new_xyz, const float* points, const float* w1, const float* bias, int C1,
                               float* pre, int* idx, int* pts_cnt, float* stats, void* workspace,
                               size_t workspace_bytes, psa_stream_t stream);

/* Fused EdgeConv, inference mode (dgcnn/models/dgcnn.py:31-47 pattern): x (b,n,c), nn_idx (b,n,k) ->
 * out (b,n,C_L) = max_j MLP([x_i, x_j - x_i]); mlp->channels[0] must equal 2c.  A single-layer MLP is evaluated as
 * (W_a - W_b).x_i + W_b.x_j: one GEMM over the b*n POINTS plus a gather-max pass (k-fold fewer FLOPs than a conv over the
 * b*n*k edges); deeper MLPs use the fused gather + MLP + max kernel.  workspace: psa_edgeconv_workspace_bytes(). */
PSA_API size_t psa_edgeconv_workspace_bytes(int b, int n, int c, int k, const psa_mlp* mlp);
PSA_API int psa_edgeconv_infer(int b, int n, int c, int k, const float* x, const int* nn_idx, const psa_mlp* mlp,
                               float* out, void* workspace, size_t workspace_bytes, psa_stream_t stream);


/* DGCNN kNN graph with the X.X^T contraction on the tensor cores and an exact refine (csrc/knn_tc.cu): same result as
 * psa_knn_graph -- indices bit-identical to the canonical fp32 evaluation (dot as an fma chain over the channels,
 * adj = (|p|^2 + (-2 dot)) + |q|^2, k smallest, lower index first on ties; dgcnn/utils/tf_util.py:638-671) -- for
 * 128 <= n <= 2048, c <= 64, k <= 32; other shapes (or a workspace smaller than psa_knn_graph_workspace_bytes) run the
 * fp32 kernel of psa_knn_graph.  workspace: bf16x3 images of the clouds, their canonical norms, the exhaustive-row worklist. */
PSA_API size_t psa_knn_graph_workspace_bytes(int b, int n, int c, int k);
PSA_API int psa_knn_graph_ws(int b, int n, int c, int k, const float* x, int* nn_idx, void* workspace, size_t workspace_bytes,
                             psa_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Training mode (SURVEY 8f rank 1): batch-statistics batch norm through every layer of a level and the
 * backward pass.  Reference semantics: pointnet2/utils/tf_util.py:155-185 (conv2d = matmul + bias, then
 * batch norm, then relu), :512-531 (tf.contrib.layers.batch_norm, is_training=True: batch mean, BIASED batch
 * variance, eps = 1e-3, moving averages updated in place with `decay`), pointnet_util.py:113-127 (MLP +
 * reduce_max), gradients tf_grouping.py:43-47 (GroupPointGrad = scatter-add by idx; index ops carry no
 * gradient, tf_sampling.py:23,58, tf_grouping.py:22,33), optimiser pointnet2/train.py:139-146 (Adam).
 * A level keeps ONE tensor per layer, the PRE-batch-norm activations y_l; everything else is recomputed
 * inside the GEMM operand loads (csrc/train_gemm.cuh).  All reductions (statistics, bias/BN gradients, weight
 * gradients, the GroupPointGrad scatter) are evaluated in a fixed order: results are bit-reproducible run to
 * run, unlike the reference's float atomicAdd scatters.
 * ------------------------------------------------------------------------------------------- */

/* Forward input of a layer: h[r][c] = relu(x[r][c] * scale[c] + shift[c]) * mask[r][c].
 * scale == NULL: identity (raw input, no relu).  mask == NULL: no dropout. */
typedef struct psa_act_in {
    const float* x;      /* (rows, ld) */
    long long ld;
    const float* scale;  /* (C) batch-norm scale = gamma / sqrt(var + eps) of the layer that produced x, or NULL */
    const float* shift;  /* (C) beta - mean * scale */
    const float* mask;   /* (rows, ld) dropout mask holding 0 or 1/keep_prob, or NULL */
    int relu;
} psa_act_in;

/* Gradient w.r.t. a layer's PRE-batch-norm output: dy[r][c] = ca[c] * dz[r][c] + cb[c] * y[r][c] + cc[c]
 * (the batch-norm backward with the batch sums folded into three per-channel constants, see
 * psa_bn_bwd_coeffs), dz = gradient w.r.t. the batch-norm output after the relu mask [y*s+t > 0]:
 *   mode 0: dz = dh[r][c] (* mask[r][c])                      dense incoming gradient
 *   mode 1: dz = dp[g][c] if argk[g][c] == r - g*pool_k and pv[g][c] > 0 else 0,  g = r / pool_k
 *           (max-pool routing: dp = gradient of the pooled output, pv = pooled value, argk = winning row).
 * ca == NULL: dy = dz (layer without batch norm).  s == NULL: no relu mask. */
typedef struct psa_grad_in {
    const float* y;      /* (rows, ld) pre-BN activations of this layer */
    long long ld;
    const float* s;      /* (C) BN scale / shift of this layer, or NULL */
    const float* t;
    int relu;
    const float* ca;     /* (C) or NULL */
    const float* cb;
    const float* cc;
    const float* dh;     /* mode 0: (rows, ld_dh) */
    long long ld_dh;
    const float* mask;   /* mode 0: dropout mask on dh, or NULL */
    const float* dp;     /* mode 1: (rows / pool_k, C) */
    const float* pv;
    const int* argk;
    int pool_k;
    int C;
    int mode;
} psa_grad_in;

/* y (rows, N) = in (rows, K) . W (K, N) + bias; stats (2, N) = per-channel [sum, sum of squares] of y (or NULL).
 * workspace: psa_train_dense_workspace_bytes(rows, K, N).  The fp32 GEMM loads psa_act_in / psa_grad_in operands element by
 * element where they are not 16-byte aligned with strides a multiple of 4.  It takes at most 65535 row tiles of 128, about
 * 8.4 M rows, in the forward (every shape the tensor-core forward does not take) and the input gradient (else
 * PSA_ERR_UNSUPPORTED, before anything is launched). */
PSA_API size_t psa_train_dense_workspace_bytes(long long rows, int K, int N);
PSA_API int psa_train_dense_fwd(long long rows, int K, int N, const psa_act_in* in, const float* W, const float* bias,
                                float* y, float* stats, void* workspace, size_t workspace_bytes, psa_stream_t stream);
/* dx (rows, K - col_skip) = dy (rows, N) . W^T restricted to input channels >= col_skip (e.g. the feature columns of a
 * concatenated [xyz, points] input; the coordinate columns come from a second product over the first rows of W). */
PSA_API int psa_train_dense_bwd_input(long long rows, int K, int N, const psa_grad_in* g, const float* W, float* dx,
                                      long long ld_dx, int col_skip, void* workspace, size_t workspace_bytes,
                                      psa_stream_t stream);
/* dW (K, N) = in^T . dy, contraction over the rows in fixed split order (deterministic). */
PSA_API int psa_train_dense_bwd_weight(long long rows, int K, int N, const psa_act_in* in, const psa_grad_in* g,
                                       float* dW, void* workspace, size_t workspace_bytes, psa_stream_t stream);

/* Pooling of (groups*pool_k, C) rows over each run of pool_k rows, the modes of pointnet_sa_module other than the fused max
 * (pointnet2/utils/pointnet_util.py:126-146): mode 0 max, 1 avg (reduce_mean), 2 weighted_avg with weights
 * exp(-5 d) / sum exp(-5 d), d = dist (groups*pool_k) = the norm of each row's centred coordinates.  out (groups, C). */
PSA_API int psa_pool_rows(long long groups, int pool_k, int C, int mode, const float* x, const float* dist, float* out,
                          psa_stream_t stream);

/* Bias gradient of a layer that is NOT followed by batch norm: db (N) = sum_r dy[r][:].  (Under batch norm the conv / fc bias
 * has an identically zero gradient -- sum_r dy = 0 -- and the training path writes exact zeros there.) */
PSA_API int psa_train_bias_grad(long long rows, int N, const psa_grad_in* g, float* db, psa_stream_t stream);

/* Training mode of psa_shared_mlp_grouped's first layer (the conv over concat([x, tile(g)]) of pointnet/models/pointnet_seg.py:81-88
 * with batch statistics).  Forward: y (rows, N) = in (rows, K) . W (K, N) + group_add[r / group_rows] + bias, and stats (2, N) of y
 * including the group term, so that batch norm sees what the conv over the concatenation produces.  One pass of the fp32 GEMM
 * behind psa_train_dense_fwd (any shape; no tensor-core path).  workspace: psa_train_dense_workspace_bytes(rows, K, N).
 * Backward: dx and dW of the rows come from psa_train_dense_bwd_input / _bwd_weight with W; the group rows' gradient is
 *   d group_add (rows / group_rows, N) = sum of dy over each group's rows  (psa_train_bias_grad_grouped),
 * whose products with W_g give dg and dW_g (psa_train_dense_bwd_input / _bwd_weight over the groups).  Under batch norm the
 * whole-batch sum of dy is zero but the per-group sums are not.  Sums in a fixed order: bit-reproducible.  group_rows must
 * divide rows (else PSA_ERR_INVALID_ARGUMENT); at most 65535 groups (else PSA_ERR_UNSUPPORTED).  psa_train_bias_grad is the
 * group_rows = rows case.  The forward takes at most 65535 row tiles of 128 (else PSA_ERR_UNSUPPORTED). */
PSA_API int psa_train_dense_fwd_grouped(long long rows, long long group_rows, int K, int N, const psa_act_in* in, const float* W,
                                        const float* bias, const float* group_add, float* y, float* stats, void* workspace,
                                        size_t workspace_bytes, psa_stream_t stream);
PSA_API int psa_train_bias_grad_grouped(long long rows, long long group_rows, int N, const psa_grad_in* g, float* db,
                                        psa_stream_t stream);

/* Batch statistics -> BN affine.  stats (2, C) sums over `count` rows; gamma, beta (C) ->
 * scale = gamma / sqrt(var + 1e-3), shift = beta - mean * scale, mean_inv (2, C) = [mean, 1/sqrt(var + eps)];
 * moving_mean / moving_var (C, may be NULL) <- decay * moving + (1 - decay) * batch  (tf_util.py:526-531). */
PSA_API int psa_bn_finalize(int C, long long count, const float* stats, const float* gamma, const float* beta,
                            float decay, float* moving_mean, float* moving_var, float* scale, float* shift,
                            float* mean_inv, psa_stream_t stream);

/* The same from the layer's output y (rows, C) itself: the mean, then the centred sum of squares, both in fp64.  For layers whose
 * output is materialised and short (the FC head, rows = batch): there the mean of a column can be large against its spread, and a
 * variance taken as E[y^2] - mean^2 from fp32 sums loses its digits. */
PSA_API int psa_bn_finalize_rows(long long rows, int C, const float* y, const float* gamma, const float* beta, float decay,
                                 float* moving_mean, float* moving_var, float* scale, float* shift, float* mean_inv,
                                 psa_stream_t stream);

/* relu(BN(y)) then max over each run of pool_k rows: pooled (groups, C), argk (groups, C) = first winning row.  A group whose
 * values are all <= 0 after the relu pools 0 with argk 0.  y, scale, shift, pooled and argk 16-byte aligned, C a multiple of 4
 * (else PSA_ERR_INVALID_ARGUMENT); the same holds for psa_pool_rows' x and out. */
PSA_API int psa_train_pool_fwd(long long groups, int pool_k, int C, const float* y, const float* scale,
                               const float* shift, float* pooled, int* argk, psa_stream_t stream);

/* Batch-norm backward sums of a layer: dbeta[c] = sum_r dz, dgamma[c] = sum_r dz * xhat (g->ca/cb/cc are ignored),
 * and the coefficients ca = gamma*inv, cb = -gamma*inv^2*dgamma/rows, cc = gamma*inv*(mean*inv*dgamma - dbeta)/rows
 * that make psa_grad_in evaluate dy.  workspace: psa_bn_bwd_workspace_bytes(C).
 * The batch-norm sums here and psa_sa_conv1_bwd / _bwd_xyz read g with 16-byte vector loads and take only such operands (else
 * PSA_ERR_INVALID_ARGUMENT): every non-NULL pointer of g they read (y, s, t, ca, cb, cc; dh and mask in mode 0; dp, pv, argk in
 * mode 1) 16-byte aligned, ld a multiple of 4 where y is read (always here, with y given), ld_dh a multiple of 4 in mode 0, and
 * in mode 1 g->C equal to the layer width (C, C1) and pool_k dividing the rows.  mean_inv here, dU of psa_sa_conv1_bwd and the
 * workspace of psa_sa_conv1_bwd_xyz are 16-byte aligned too. */
PSA_API size_t psa_bn_bwd_workspace_bytes(int C);
PSA_API int psa_bn_bwd_coeffs(long long rows, int C, const psa_grad_in* g, const float* gamma, const float* mean_inv,
                              float* dgamma, float* dbeta, float* ca, float* cb, float* cc, void* workspace,
                              size_t workspace_bytes, psa_stream_t stream);

/* Backward of the fused first layer of a set-abstraction level (psa_sa_conv1_prebn): with dy0 = g over the
 * b*m*nsample grouped rows,  dW_xyz (3, C1) = sum_r (xyz[idx_r] - new_xyz[q_r])^T dy0[r]  and, if dU != NULL,
 * dU (b*n, C1) = GroupPointGrad(dy0, idx) (tf_grouping_g.cu:61-78) as a stable counting sort of the (row -> point)
 * entries followed by an ordered gather (each source point adds its rows in ascending row order: deterministic).  The feature part of the layer then is two dense products on the b*n
 * POINTS: dpoints = dU . W1[3:]^T and dW1[3:] = points^T . dU.  workspace: psa_sa_conv1_bwd_workspace_bytes(...). */
PSA_API size_t psa_sa_conv1_bwd_workspace_bytes(int b, int n, int m, int nsample, int C1, int want_dU);
PSA_API int psa_sa_conv1_bwd(int b, int n, int m, int nsample, int C1, const float* xyz, const float* new_xyz,
                             const int* idx, const psa_grad_in* g, float* dW_xyz, float* dU, void* workspace,
                             size_t workspace_bytes, psa_stream_t stream);

/* Coordinate gradient of the fused first layer (the reference's GroupPointGrad of grouped_xyz plus the "- tile(new_xyz)" term,
 * pointnet_util.py:40-46, tf_grouping.py:43-47).  With dy0 = g over the b*m*nsample grouped rows (the same psa_grad_in as
 * psa_sa_conv1_bwd) and W_xyz (3, C1) = the coordinate rows of the first weight (16-byte aligned), every row r = (cloud, q, k) gives
 * v_r = W_xyz . dy0_r, and
 *   dxyz (b, n, 3)     = sum over the rows r with idx_r = p of v_r, each point's rows added in ascending row order (stable
 *                        counting sort of idx, as in psa_sa_conv1_bwd's dU);
 *   dnew_xyz (b, m, 3) = -(v_{q,0} + v_{q,1} + ...), added in slot order.
 * Padding rows (copies of slot 0) and empty balls (idx = 0) are rows like any other.  The gradient with respect to the input
 * cloud is dxyz + GatherPointGrad(dnew_xyz + whatever else new_xyz receives, fps_idx) (psa_gather_point_grad).  Both outputs are
 * fully written; no float atomics, every sum in a fixed order: bit-reproducible.  C1 a multiple of 4, at most 1024 (else
 * PSA_ERR_UNSUPPORTED).  workspace: psa_sa_conv1_bwd_xyz_workspace_bytes(...). */
PSA_API size_t psa_sa_conv1_bwd_xyz_workspace_bytes(int b, int n, int m, int nsample);
PSA_API int psa_sa_conv1_bwd_xyz(int b, int n, int m, int nsample, int C1, const float* W_xyz, const int* idx, const psa_grad_in* g,
                                 float* dxyz, float* dnew_xyz, void* workspace, size_t workspace_bytes, psa_stream_t stream);

/* Training-mode single-layer EdgeConv (dgcnn/models/dgcnn.py:41-47, dgcnn/utils/tf_util.py:115-173,462-499):
 *   out_ic = max_j relu(BN(y_ij)),  y_ij = [x_i, x_j - x_i] . W + bias,  BN with the batch statistics of all b*n*k edges.
 * Replaces get_edge_feature (tf_util.py:674-706) + conv2d + batch_norm(is_training=True) + relu + reduce_max and their gradients
 * without any (b,n,k,.) tensor: with Q = x (W_a - W_b) + bias and P = x W_b (W_a = rows 0..c of W, W_b = rows c..2c), every
 * edge value is y_ij = Q_i + P_nn(i,j), recomputed from the (b*n, 2 C_out) buffer PQ = [Q | P] in every pass.  x (b,n,c),
 * nn_idx (b,n,k) int32 with within-cloud indices in [0, n), W (2c, C_out), bias (C_out) or NULL.  C_out a multiple of 32,
 * at most 256 (else PSA_ERR_UNSUPPORTED); any c >= 1, k >= 1; the backward takes n <= 51200.  One workspace serves the three
 * calls: psa_edgeconv_train_workspace_bytes() bytes, 256-byte aligned.  Every reduction runs in a fixed order: bit-reproducible.
 *
 * forward 1: PQ (b*n, 2 C_out) and stats (2, C_out) = per-channel [sum y, sum y^2] over the edges; then psa_bn_finalize with
 *            count = b*n*k gives scale, shift, mean_inv and updates the moving averages.  stats == NULL: PQ only, for frozen batch
 *            norm (inference mode: scale = gamma / sqrt(moving_var + 1e-3), shift = beta - moving_mean * scale, computed by the
 *            caller), whose backward is psa_edgeconv_frozen_bwd. */
PSA_API size_t psa_edgeconv_train_workspace_bytes(int b, int n, int c, int k, int C_out);
PSA_API int psa_edgeconv_train_fwd(int b, int n, int c, int k, int C_out, const float* x, const int* nn_idx, const float* W,
                                   const float* bias, float* PQ, float* stats, void* workspace, size_t workspace_bytes,
                                   psa_stream_t stream);
/* forward 2: pooled (b*n, C_out) = max_j relu(y_ij * scale + shift) and ties (b*n, C_out) = how many edges reach that maximum
 * bit for bit -- uint8 when k <= 255, int32 otherwise. */
PSA_API int psa_edgeconv_train_pool(int b, int n, int k, int C_out, const int* nn_idx, const float* PQ, const float* scale,
                                    const float* shift, float* pooled, void* ties, psa_stream_t stream);
/* backward: dout (b*n, C_out) = gradient of pooled, split evenly among the tied edges of a positive maximum (torch.amax / TF
 * reduce_max) -> dW (2c, C_out), dgamma, dbeta (C_out), dx (b*n, c).  The conv bias under batch norm has an exactly zero
 * gradient (not written).  The kNN graph carries no gradient.  scale, shift, gamma, mean_inv as the forward used them. */
PSA_API int psa_edgeconv_train_bwd(int b, int n, int c, int k, int C_out, const float* x, const int* nn_idx, const float* W,
                                   const float* PQ, const float* scale, const float* shift, const float* gamma,
                                   const float* mean_inv, const float* pooled, const void* ties, const float* dout, float* dW,
                                   float* dgamma, float* dbeta, float* dx, void* workspace, size_t workspace_bytes,
                                   psa_stream_t stream);
/* backward with frozen batch norm (after psa_edgeconv_train_fwd with stats == NULL and psa_edgeconv_train_pool on the frozen
 * scale / shift): dout routed to the tied edges of a positive maximum as above, dy = scale * dz -> dx (b*n, c) only; no
 * batch-norm sums and no variable gradients.  Same limits and workspace as psa_edgeconv_train_bwd. */
PSA_API int psa_edgeconv_frozen_bwd(int b, int n, int c, int k, int C_out, const float* x, const int* nn_idx, const float* W,
                                    const float* PQ, const float* scale, const float* shift, const float* pooled, const void* ties,
                                    const float* dout, float* dx, void* workspace, size_t workspace_bytes, psa_stream_t stream);

/* Training mode of a two-layer EdgeConv (DGCNN's input transform net, transform_nets.py:18-27): out_ic = max_j relu(BN2(relu(BN1(
 * [x_i, x_j - x_i] . W1 + b1)) . W2 + b2)), both batch norms with batch statistics over all E = b*n*k edges.  No per-edge tensor
 * is stored in the forward; the backward keeps one, the (E, C1) gradient of layer 1.  Layer 1 is the single-layer op above:
 * psa_edgeconv_train_fwd with C_out = C1 gives PQ (b*n, 2 C1) and its statistics, psa_bn_finalize(C1, E, ...) its affine.  C1 = 64,
 * C2 = 128 and k <= 32 (else PSA_ERR_UNSUPPORTED); any c >= 1; the backward takes n <= 51200.  One workspace of
 * psa_edgeconv2_train_workspace_bytes() bytes, 256-byte aligned, serves all calls including the layer-1 forward.  The per-edge
 * products run on the tensor cores (three bf16 pieces per operand); every reduction runs in a fixed order: bit-reproducible.
 *
 * forward: stats2 (2, C2) = per-channel [sum y2, sum y2^2] over the edges; then psa_bn_finalize(C2, E, ...). */
PSA_API size_t psa_edgeconv2_train_workspace_bytes(int b, int n, int c, int k, int C1, int C2);
PSA_API int psa_edgeconv2_train_fwd(int b, int n, int c, int k, int C1, int C2, const int* nn_idx, const float* PQ,
                                    const float* scale1, const float* shift1, const float* W2, const float* bias2, float* stats2,
                                    void* workspace, size_t workspace_bytes, psa_stream_t stream);
/* pool: pooled (b*n, C2) = max_j relu(y2_ij * scale2 + shift2); mask (b*n, C2) = bit j set for every edge that reaches the
 * maximum bit for bit; ywin (b*n, C2) = y2 of the first of them (pre batch norm). */
PSA_API int psa_edgeconv2_train_pool(int b, int n, int c, int k, int C1, int C2, const int* nn_idx, const float* PQ,
                                     const float* scale1, const float* shift1, const float* W2, const float* bias2,
                                     const float* scale2, const float* shift2, float* pooled, unsigned int* mask, float* ywin,
                                     void* workspace, size_t workspace_bytes, psa_stream_t stream);
/* backward: dout (b*n, C2) = gradient of pooled, split evenly among the masked edges of a positive maximum -> dW1 (2c, C1),
 * dgamma1, dbeta1 (C1), dW2 (C1, C2), dgamma2, dbeta2 (C2), dx (b*n, c).  Both conv biases have exactly zero gradient under
 * batch norm (not written); the kNN graph carries no gradient. */
PSA_API int psa_edgeconv2_train_bwd(int b, int n, int c, int k, int C1, int C2, const float* x, const int* nn_idx,
                                    const float* W1, const float* PQ, const float* scale1, const float* shift1,
                                    const float* gamma1, const float* mean_inv1, const float* W2, const float* bias2,
                                    const float* gamma2, const float* mean_inv2, const float* pooled, const unsigned int* mask,
                                    const float* ywin, const float* dout, float* dW1, float* dgamma1, float* dbeta1, float* dW2,
                                    float* dgamma2, float* dbeta2, float* dx, void* workspace, size_t workspace_bytes,
                                    psa_stream_t stream);
/* Frozen batch norm (inference mode) in both layers: the forward is psa_edgeconv_train_fwd with stats == NULL followed by
 * psa_edgeconv2_train_pool on the frozen scale1 / shift1 / scale2 / shift2 (no psa_edgeconv2_train_fwd).  backward: dout routed
 * to the masked edges of a positive maximum, dy2 = scale2 * dz2, dy1 = scale1 * dz1 -> dx (b*n, c) only; no batch-norm sums and
 * no variable gradients.  pooled, mask, ywin as the pool wrote them; bias2 may be NULL.  Same limits and workspace as
 * psa_edgeconv2_train_bwd. */
PSA_API int psa_edgeconv2_frozen_bwd(int b, int n, int c, int k, int C1, int C2, const float* x, const int* nn_idx,
                                     const float* W1, const float* PQ, const float* scale1, const float* shift1, const float* W2,
                                     const float* bias2, const float* scale2, const float* pooled, const unsigned int* mask,
                                     const float* ywin, const float* dout, float* dx, void* workspace, size_t workspace_bytes,
                                     psa_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * SpiderCNN, inference mode (SpiderCNN/utils/tf_util.py:127-235 spiderConv, :363-377 topk_pool,
 * :407-429 group_norm_for_conv)
 * ------------------------------------------------------------------------------------------- */

/* One spiderConv layer up to its group norm, without the (b,n,k,c*T) product tensor of the reference:
 *   y[p][o] = bias[o] + sum_j sum_c sum_t  h[nn(p,j)][c] * g_t(delta[p][j]) * W[j][c*T + t][o]
 *   h = relu(feat * feat_scale[b][c] + feat_shift[b][c])   (the previous layer's group norm + ReLU, per cloud b),
 *       or feat itself when feat_scale == NULL (no ReLU: the first layer reads the coordinates);
 *   g_t(d) = sum_m taylor[m][t] * mono_m(d) over the 20 monomials of degree <= 3, in the order of the reference's
 *       variables: x, y, z, xyz, xy, yz, xz, 1 (`biases`), xx, yy, zz, xxy, xyy, xxz, xzz, yyz, yzz, xxx, yyy, zzz.
 * delta (b,n,k,3) = group_point(xyz, nn_idx) - xyz; nn_idx (b,n,k) int32 in [0, n); feat (b,n,c); feat_scale,
 * feat_shift (b,c) or NULL; taylor (20,T); W (k, c*T, c_out) = the [1,k] conv's kernel; bias (c_out) -> y (b,n,c_out),
 * pre-group-norm.  The conv runs as one GEMM over the b*n points whose operand is gathered and scaled while it is
 * staged (tensor cores for b*n >= 128, c % 32 == 0, k*c*T % 64 == 0, c_out == 64 or c_out % 128 == 0, feat 16-byte
 * aligned and feat_scale / feat_shift / bias / y 8-byte aligned; the fp32-FMA kernel otherwise and in mode 1; the arithmetic
 * modes of psa_set_mlp_mode apply).  1 <= k <= 32.  workspace: psa_spider_conv_workspace_bytes(), sized for the tensor path
 * whenever the dims allow it, 256-byte aligned. */
PSA_API size_t psa_spider_conv_workspace_bytes(int b, int n, int c, int k, int T, int c_out);
PSA_API int psa_spider_conv_infer(int b, int n, int c, int k, int T, int c_out, const float* delta, const int* nn_idx,
                                  const float* feat, const float* feat_scale, const float* feat_shift, const float* taylor,
                                  const float* W, const float* bias, float* y, void* workspace, size_t workspace_bytes,
                                  psa_stream_t stream);

/* Group norm of y (b,n,c) as a per-cloud affine: `groups` contiguous channel groups (groups divides c); per (cloud, group)
 * the mean and then the centred variance (biased) over the group's channels and the n points, both in fp64 ->
 * scale[b][ch] = gamma[ch] / sqrt(var + eps), shift[b][ch] = beta[ch] - mean * scale.  out (b,n,c) or NULL:
 * y * scale + shift, then a ReLU if relu != 0. */
PSA_API int psa_group_norm_affine(int b, int n, int c, int groups, float eps, const float* y, const float* gamma,
                                  const float* beta, float* scale, float* shift, float* out, int relu, psa_stream_t stream);

/* tf.nn.top_k over the points of h = y * scale + shift (+ ReLU if relu != 0; scale == NULL: h = y), k == 2:
 * y (b,n,c), scale, shift (b,c) -> out[b][offset + ch][r] of out (b, out_channels, 2), r = 0 the largest.  n >= 2. */
PSA_API int psa_topk_pool(int b, int n, int c, int k, const float* y, const float* scale, const float* shift, int relu,
                          float* out, int out_channels, int offset, psa_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * SpiderCNN, training backward (fp32 FMA, no float atomics: every sum in a fixed order).  Notation of
 * psa_spider_conv_infer; dy (b,n,c_out) = the gradient of a layer's pre-group-norm output y.  T == 5 only
 * (SpiderCNN's taylor_channel), else PSA_ERR_UNSUPPORTED.  No (b,n,k,c*T) tensor is formed.
 * ------------------------------------------------------------------------------------------- */

/* g (b,n,k,T) = the Taylor filter values g_t(delta[p][j]) of psa_spider_conv_infer, bit-identical to its own. */
PSA_API int psa_spider_taylor_filter(int b, int n, int k, int T, const float* delta, const float* taylor, float* g,
                                     psa_stream_t stream);

/* Scratch of psa_spider_conv_bwd_weight, psa_spider_taylor_grad and psa_spider_gn_bwd for these dims (one buffer serves all
 * three); 256-byte aligned.  0 for dims none of them takes. */
PSA_API size_t psa_spider_conv_bwd_workspace_bytes(int b, int n, int c, int k, int T, int c_out);

/* dW (k, c*T, c_out) = A^T . dy with A[p][j*c*T + ch*T + t] = h[nn(p,j)][ch] * g[p][j][t] (the reference's conv-input row
 * order, so dW is the variable's gradient as it is laid out); h as in psa_spider_conv_infer. */
PSA_API int psa_spider_conv_bwd_weight(int b, int n, int c, int k, int T, int c_out, const int* nn_idx, const float* feat,
                                       const float* feat_scale, const float* feat_shift, const float* g, const float* dy, float* dW,
                                       void* workspace, size_t workspace_bytes, psa_stream_t stream);

/* With Q[p][j][ch][t] = sum_o dy[p][o] * W[j][ch*T + t][o] (never stored):
 *   D (b,n,k,c)  D[p][j][ch] = sum_t g[p][j][t] * Q     (NULL: skipped; psa_group_point_grad(D, nn_idx) is then dh of feat)
 *   dg (b,n,k,T) dg[p][j][t] = sum_ch h[nn(p,j)][ch] * Q */
PSA_API int psa_spider_conv_bwd_data(int b, int n, int c, int k, int T, int c_out, const int* nn_idx, const float* feat,
                                     const float* feat_scale, const float* feat_shift, const float* g, const float* W, const float* dy,
                                     float* D, float* dg, psa_stream_t stream);

/* dtaylor[m * ld_taylor + t] = sum_{p,j} dg[p][j][t] * mono_m(delta[p][j]), m in psa_spider_conv_infer's monomial order,
 * accumulated in fp64. */
PSA_API int psa_spider_taylor_grad(int b, int n, int k, int T, const float* delta, const float* dg, float* dtaylor, int ld_taylor,
                                   void* workspace, size_t workspace_bytes, psa_stream_t stream);

/* Backward of h = relu(group_norm(y)) and of its top-2 pooling: per (cloud, group) the forward's fp64 mean and variance
 * (psa_group_norm_affine), the winners of psa_topk_pool on relu(y * scale + shift) with tf.nn.top_k's tie order (lower point
 * first), dh = dpool routed to the winners (dpool (b, pool_channels, 2), this layer's channels at offset) + dh_next (b,n,c) or
 * NULL, dz = dh where y * scale + shift > 0, and
 *   dy = rstd * (gamma dz - mean_group(gamma dz) - xhat * mean_group(gamma dz xhat)),  dgamma = sum dz xhat,  dbeta = sum dz.
 * c / groups must divide 256; n >= 2. */
PSA_API int psa_spider_gn_bwd(int b, int n, int c, int groups, float eps, const float* y, const float* scale, const float* shift,
                              const float* gamma, const float* dpool, int pool_channels, int offset, const float* dh_next, float* dy,
                              float* dgamma, float* dbeta, void* workspace, size_t workspace_bytes, psa_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * 3DmFV-Net, inference mode (3DmFV-Net/utils/tf_util.py:578-652 get_3dmfv, :254-311 conv3d, :406-429 pools)
 * Grid activations are (b * r^3, c) in voxel-major row order: row = voxel * b + cloud, voxel = (d * r + h) * r + w.
 * ------------------------------------------------------------------------------------------- */

/* The modified Fisher vector of get_3dmfv(flatten=False) before its final transpose: points (b,n,3), w (G), mu (G,3), sigma
 * (G,3) (standard deviations) -> out (b,G,20), columns [d_pi max, sum | d_mu max xyz, min xyz, sum xyz | d_sigma max xyz, min
 * xyz, sum xyz], power- (sign(v) |v|^0.5) and L2-normalised over the G Gaussians per (cloud, column).  The soft assignment is
 * evaluated in the log domain, log w - sum_d log sigma - |z|^2 / 2 shifted by its maximum over the Gaussians: where the
 * reference's fp32 densities all underflow it returns NaN, this op the finite limit.  Terms and sums in fp64, every reduction
 * in a fixed order (bit-identical reruns), no (b,n,G) buffer.  One block per cloud; PSA_ERR_UNSUPPORTED when n and G do not fit
 * its shared memory (about 8 * (2n + 27G) + 12n bytes <= 220 KB). */
PSA_API int psa_fisher_vector(int b, int n, int G, const float* points, const float* w, const float* mu, const float* sigma,
                              float* out, psa_stream_t stream);

/* One tf_util.conv3d layer on an r^3 grid, SAME padding, stride 1, k in {1, 3, 5}: x rows (b*r^3) of stride ldx, c channels;
 * W = the TF kernel (k,k,k,c,c_out), read as a (k^3 c, c_out) matrix; out[row * ldo + o] = relu?((x * W)[row][o] * scale[o] +
 * shift[o]) (scale NULL: + shift only), the folded bias and batch norm.  The row strides let each inception branch read and
 * write its slice of the concatenated output in place.  Tensor cores for c % 64 == 0, c_out % 32 == 0, x 16-byte aligned with
 * ldx % 4 == 0, out 8-byte aligned with ldo even and scale / shift 8-byte aligned (a tile issues no MMA for a tap outside the
 * grid for all its rows; the tap loop is split across CTAs and the partials added in a fixed order), the fp32-FMA kernel
 * otherwise and in mode 1; the arithmetic modes of psa_set_mlp_mode apply.  workspace: psa_conv3d_workspace_bytes() queried
 * in the mode of the call (0 when the shape or the mode takes the FMA kernel), 256-byte aligned. */
PSA_API size_t psa_conv3d_workspace_bytes(int b, int r, int k, int c, int c_out);
PSA_API int psa_conv3d_infer(int b, int r, int k, int c, int c_out, const float* x, long long ldx, const float* W,
                             const float* scale, const float* shift, int relu, float* out, long long ldo, void* workspace,
                             size_t workspace_bytes, psa_stream_t stream);

/* The inception module's pools on voxel-major rows x (b*r^3, c): kind 0 = SAME 3^3 average, stride 1, divided by the number
 * of in-grid cells -> (b*r^3, c); kind 1 = SAME 2^3 max, stride 2, padded at the far end -> (b*ceil(r/2)^3, c). */
PSA_API int psa_pool3d(int b, int r, int c, int kind, const float* x, float* out, psa_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * 3DmFV-Net, training (3DmFV-Net/train.py:163-173: the Fisher vector takes fed placeholders, so the backward stops at the
 * grid).  fp32 FMA in every arithmetic mode, no float atomics: every sum runs in a fixed order and a step is bit-reproducible.
 * Notation of psa_conv3d_infer; K = k^3 * c; dy (b*r^3, c_out) contiguous = the gradient of a conv's pre-batch-norm output.
 * Neither product forms the (b*r^3, K) im2col operand, and both skip every 16-wide contraction block for which each kernel tap
 * it touches lies outside the grid for all the rows it touches.
 * ------------------------------------------------------------------------------------------- */

/* Scratch of psa_conv3d_bwd_weight and psa_conv3d_bwd_data (split-contraction partials), 256-byte aligned; 0 for bad dims. */
PSA_API size_t psa_conv3d_bwd_workspace_bytes(int b, int r, int k, int c, int c_out);

/* dW (K, c_out) = A^T . dy, A[row][(tap, ch)] = x[neighbour(row, tap)][ch] or 0 outside the grid: the gradient of the TF kernel
 * (k,k,k,c,c_out) in its own layout.  Split over the rows, partials added in split order.  x rows of stride ldx. */
PSA_API int psa_conv3d_bwd_weight(int b, int r, int k, int c, int c_out, const float* x, long long ldx, const float* dy, float* dW,
                                  void* workspace, size_t workspace_bytes, psa_stream_t stream);

/* dx[u][ch] (+)= sum_tap sum_o dy[u - offset(tap)][o] * W[tap][ch][o] (terms outside the grid are 0): the gradient of the conv's
 * input, written at row stride ld_dx; accumulate != 0 adds it to what dx holds.  Split over the taps, partials added in split
 * order. */
PSA_API int psa_conv3d_bwd_data(int b, int r, int k, int c, int c_out, const float* dy, const float* W, float* dx, long long ld_dx,
                                int accumulate, void* workspace, size_t workspace_bytes, psa_stream_t stream);

/* The multiply-adds the two products issue at these dims (their tiles and skip rule, no GPU needed) and the multiply-adds whose
 * tap lies inside the grid: issued_weight, issued_data, in_grid (each may be NULL). */
PSA_API int psa_conv3d_bwd_macs(int b, int r, int k, int c, int c_out, long long* issued_weight, long long* issued_data,
                                long long* in_grid);

/* out[row * ldo + ch] = relu(y[row][ch] * scale[ch] + shift[ch]) (one fmaf, the gate psa_grad_in tests): y (rows, C). */
PSA_API int psa_mfv_bn_relu(long long rows, int C, const float* y, const float* scale, const float* shift, float* out, long long ldo,
                            psa_stream_t stream);

/* dy (rows, C) = the psa_grad_in g evaluated at every element (mode 0), materialised for the conv3d products' gathers. */
PSA_API int psa_mfv_bn_dy(long long rows, int C, const psa_grad_in* g, float* dy, psa_stream_t stream);

/* psa_pool3d's SAME 2^3 stride-2 max that also records its winner: winner[v][ch] = the first maximum in window order
 * (dz, dy, dx) as dz * 4 + dy * 2 + dx; cells of the far-end padding never win.  out, winner (b*ceil(r/2)^3, c). */
PSA_API int psa_pool3d_max_train(int b, int r, int c, const float* x, float* out, unsigned char* winner, psa_stream_t stream);

/* Backward of psa_pool3d: dout (b*ro^3, c) -> dx (b*r^3, c), every element written.  kind 0 (3^3 average): dx[u] = sum over the
 * windows v holding u, in (dz, dy, dx) order, of dout[v] / count(v).  kind 1 (2^3 max): dx[u] = dout[v] where u is v's recorded
 * winner, else 0. */
PSA_API int psa_pool3d_bwd(int b, int r, int c, int kind, const float* dout, const unsigned char* winner, float* dx,
                           psa_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * PointCNN, inference mode (PointCNN/pointcnn.py:10-52 xconv, pointfly.py:122-128, 163-176 knn_indices_general,
 * :298-347 dense / conv2d / depthwise_conv2d / separable_conv2d).  Every layer with batch norm has no bias and applies
 * ELU before the batch norm: a = elu(x . W) * s + t, s = gamma / sqrt(moving_variance + 1e-3), t = beta - moving_mean * s.
 * ------------------------------------------------------------------------------------------- */

/* knn_indices_general(queries, points, k*d, sort=True) followed by indices[:, :, ::d] (pointcnn.py:12-13): points (b,n,3),
 * queries (b,m,3) -> idx (b,m,k) int32 in [0, n).  D = (|q|^2 + (-2 q.p)) + |p|^2 with the dot and the norms fma chains over
 * x, y, z from 0 (the order of oracle/psa_oracle.c:orc_dgcnn_knn); the k*d smallest in ascending order, lower index first on
 * ties (tf.nn.top_k), then every d-th entry from the first.  Duplicate points stay in the lists: the reference's unique=True
 * (pointfly.py:142-144) adds to a local name only.  k*d <= 64 and k*d <= n. */
PSA_API int psa_knn_dilated(int b, int n, int m, int k, int d, const float* points, const float* queries, int* idx,
                            psa_stream_t stream);

/* The weights of one X-Conv layer in TF's layouts, each with its batch norm as (s, t):
 *   w_pts0 (3, c_pts)        `<tag>nn_fts_from_pts_0/kernel`     w_pts1 (c_pts, c_pts)  `<tag>nn_fts_from_pts/kernel`
 *   w_x0   (1, K, 3, K*K)    `<tag>X_0/kernel`                   w_x1, w_x2 (1, K, K, K) `<tag>X_1/depthwise_weights`, X_2
 *   w_dw   (1, K, c_in, dm)  `<tag>fts_conv/depthwise_kernel`, c_in = c_pts + c_prev.  X_2 has no ELU (pointcnn.py:37). */
typedef struct psa_xconv {
    int K, c_pts, c_prev, dm;
    const float *w_pts0, *s_pts0, *t_pts0;
    const float *w_pts1, *s_pts1, *t_pts1;
    const float *w_x0, *s_x0, *t_x0;
    const float *w_x1, *s_x1, *t_x1;
    const float *w_x2, *s_x2, *t_x2;
    const float* w_dw;
} psa_xconv;

/* One X-Conv layer up to the depthwise stage of its separable conv, per query (pointcnn.py:15-44):
 *   local[j] = pts[idx[j]] - q;  lifted = dense(dense(local)) (K, c_pts);  F = [lifted | fts[idx[j]]] (K, c_in);
 *   X0[a*K + b] = sum_{j,d} local[j][d] w_x0[j][d][a*K + b] (ELU, BN);  X1[b*K + m] = sum_a X0[a*K + b] w_x1[a][b][m] (ELU, BN);
 *   X2 likewise from X1 with w_x2 (BN, no ELU);  fts_X[i][c] = sum_j X2[i*K + j] F[j][c];
 *   out[c*dm + m] = sum_i fts_X[i][c] w_dw[i][c][m].
 * pts (b,n,3), qrs (b,P,3), idx (b,P,K) int32 in [0, n), fts (b,n,c_prev) or NULL when c_prev == 0 -> out (b*P, c_in*dm).
 * fp32 FMA, one tile of queries per block in shared memory: no (b,P,K,.) tensor reaches global memory.  1 <= K <= 16. */
PSA_API int psa_xconv_core(int b, int n, int P, const float* pts, const float* qrs, const int* idx, const float* fts,
                           const psa_xconv* layer, float* out, psa_stream_t stream);

/* out[row * ldo + o] = elu((x . W)[row][o] + bias[o]) * scale[o] + shift[o] for o < N: x rows of stride ldx, K channels; W (K, N);
 * bias (N) or NULL.  The row strides let a layer write its slice of a wider row (the global branch and the pointwise conv of
 * the last X-Conv layer, pointcnn.py:47-50).  Tensor cores for rows >= 128, K % 4 == 0, ldx % 4 == 0 and x 16-byte aligned:
 * the operand columns past K read as zero up to a multiple of 64, W is padded to 64-wide column blocks (taken 128 wide when
 * their count is even) and only the N real columns are written; the fp32-FMA kernel otherwise and in mode 1.  The arithmetic
 * modes of psa_set_mlp_mode apply.  workspace: psa_dense_elu_affine_workspace_bytes() queried in the mode of the call (0 when
 * the dims or the mode take the FMA kernel), 256-byte aligned. */
PSA_API size_t psa_dense_elu_affine_workspace_bytes(long long rows, int K, int N);
PSA_API int psa_dense_elu_affine(long long rows, int K, int N, const float* x, long long ldx, const float* W, const float* bias,
                                 const float* scale, const float* shift, float* out, long long ldo, void* workspace,
                                 size_t workspace_bytes, psa_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * PointCNN, training mode (PointCNN/pointcnn.py:10-52, pointfly.py:298-347 with is_training=True; train.py:138-164).  Every
 * batch norm takes the statistics of its batch: a layer BN(elu(z)) keeps only a = elu(z) (z itself for X_2, which has no ELU),
 * and the next layer applies the batch's (s, t) to a.  fp32 FMA in every arithmetic mode, no float atomics: weight gradients
 * are summed per block over a fixed set of tiles and the block partials added in block order, so a step is bit-reproducible.
 * Notation of psa_xconv_core; R = b*P queries.
 * ------------------------------------------------------------------------------------------- */

/* The activations a training forward saves per X-Conv layer, every one contiguous:
 *   local (R*K, 3) = pts[idx] - q;  a_p0, a_p1 (R*K, c_pts) the two lifting layers;  a_x0, a_x1, a_x2 (R, K*K) X_0, X_1, X_2. */
typedef struct psa_xconv_saved {
    float* local;
    float* a_p0;
    float* a_p1;
    float* a_x0;
    float* a_x1;
    float* a_x2;
} psa_xconv_saved;

/* One forward stage of an X-Conv layer, each pre-batch-norm value evaluated with psa_xconv_core's own fmaf chain, so that
 * psa_xconv_core run with the batch (s, t) of the five layers in `layer` computes its output from exactly these activations:
 *   stage 0: local, a_p0 = elu(local . w_pts0), a_x0 = elu(local (R, 3K) . w_x0)
 *   stage 1: a_p1 = elu(BN(a_p0) . w_pts1), a_x1 = elu(depthwise(BN(a_x0), w_x1))   BN(a) = a * s + t with layer's s_pts0 / s_x0 ...
 *   stage 2: a_x2 = depthwise(BN(a_x1), w_x2)
 * pts (b,n,3), qrs (b,P,3), idx (b,P,K) as psa_xconv_core takes them; the (s, t) a stage does not read may be NULL. */
PSA_API int psa_xconv_train_stage(int stage, int b, int n, int P, const float* pts, const float* qrs, const int* idx,
                                  const psa_xconv* layer, const psa_xconv_saved* saved, psa_stream_t stream);

/* Scratch of psa_xconv_train_bwd_top and psa_xconv_depthwise_bwd for one layer (block partials); 0 for dims they do not take. */
PSA_API size_t psa_xconv_train_bwd_workspace_bytes(int b, int P, int K, int c_pts, int c_prev, int dm);

/* Backward of the core's top from d_dw (R, c_in*dm), the gradient of psa_xconv_core's output: with X2n = BN(a_x2) (K, K),
 * F = [BN(a_p1) | fts[idx]] (K, c_in) and fts_X = X2n . F recomputed per query,
 *   dW_dw (K, c_in, dm) = sum_queries fts_X[i][c] d_dw[c*dm + m];  d fts_X[i][c] = sum_m d_dw[c*dm + m] w_dw[i][c][m];
 *   dX2n (R, K*K) = d fts_X . F^T;  dF = X2n^T . d fts_X, written as dF_lift (R*K, c_pts) and dF_prev (R*K, c_prev).
 * fts and dF_prev are given exactly when c_prev > 0; psa_group_point_grad(b, n, c_prev, P, K, dF_prev, idx, ...) turns dF_prev
 * into the gradient of fts.  Reads layer's s_pts1, t_pts1, s_x2, t_x2, w_dw and saved's a_p1, a_x2. */
PSA_API int psa_xconv_train_bwd_top(int b, int n, int P, const int* idx, const float* fts, const psa_xconv* layer,
                                    const psa_xconv_saved* saved, const float* d_dw, float* dX2n, float* dF_lift, float* dF_prev,
                                    float* dW_dw, void* workspace, size_t workspace_bytes, psa_stream_t stream);

/* Backward of a depthwise X layer z[b*K + m] = sum_a x[a*K + b] W[a][b][m] over R rows, x = a_in * s + t (a_in (R, K*K)):
 *   dz = g evaluated per element (mode 0: the batch-norm backward of the layer's output, g->y its saved activations), times
 *        TF's EluGrad (g->y < 0 ? g->y + 1 : 1) when elu != 0;
 *   dW (K, K, K) = sum_r x[a*K + b] dz[b*K + m];  dx (R, K*K) = sum_m dz[b*K + m] W[a][b][m], the gradient of x.
 * workspace: psa_xconv_train_bwd_workspace_bytes of the layer. */
PSA_API int psa_xconv_depthwise_bwd(long long rows, int K, const float* x, const float* s, const float* t, const psa_grad_in* g, int elu,
                                    const float* W, float* dW, float* dx, void* workspace, size_t workspace_bytes, psa_stream_t stream);

/* dz (rows, C) = g (mode 0) evaluated at every element times TF's EluGrad on g->y: the gradient of z for a layer BN(elu(z)),
 * materialised for the dense products (psa_train_dense_bwd_weight / _bwd_input with a plain psa_grad_in over dz). */
PSA_API int psa_elu_bn_dy(long long rows, int C, const psa_grad_in* g, float* dz, psa_stream_t stream);

/* out[r * ldo + c] = a[r][c] * s[c] + t[c] (one fmaf): a (rows, C) contiguous, the batch norm of a layer written into its slice of
 * a wider row. */
PSA_API int psa_bn_affine_rows(long long rows, int C, const float* a, const float* s, const float* t, float* out, long long ldo,
                               psa_stream_t stream);

/* Mean sparse softmax cross-entropy (pointnet2_cls_ssg.py:50-57) and its gradient: logits (b, c), labels (b) int32 ->
 * loss (1), dlogits (b, c) = (softmax - onehot) / b. */
PSA_API int psa_softmax_xent(int b, int c, const float* logits, const int* labels, float* loss, float* dlogits,
                             psa_stream_t stream);

/* tf.train.AdamOptimizer step over one flat parameter vector (pointnet2/train.py:139-146):
 * g = grad * grad_scale; m = b1 m + (1-b1) g; v = b2 v + (1-b2) g^2; p -= lr sqrt(1-b2^t)/(1-b1^t) m / (sqrt(v) + eps). */
PSA_API int psa_adam_step(long long count, float* params, const float* grads, float* m, float* v, float lr, float beta1,
                          float beta2, float eps, int step, float grad_scale, psa_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* PSA_H_ */
