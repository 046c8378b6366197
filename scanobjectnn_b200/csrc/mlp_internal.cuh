// mlp_internal.cuh -- pieces of mlp.cu shared with tc_mlp.cu
#pragma once
#include "common.cuh"

namespace psa {

struct DenseArgs {
    long long rows;
    int K, N;
    int pool_k;          // 1 = none
    int relu;
    const float* x;      // (rows, K)
    const float* W;      // (K, N)
    const float* scale;  // (N) or null
    const float* shift;  // (N)
    float* out;          // (rows, N) or (rows/pool_k, N)
    // optional per-row-group input, pool_k == 1 only: row r adds group_add[r / group_rows] (N) to x . W before the affine
    const float* group_add = nullptr;
    long long group_rows = 0;
    // optional side input, pool_k == 1 only: row r adds xyz3[r] (3) . w3 (3, N) to x . W before the affine
    const float* xyz3 = nullptr;
    const float* w3 = nullptr;
};


int launch_dense(const DenseArgs& d, cudaStream_t st);
size_t fc_small_workspace_bytes(int K, int N);
int launch_fc_small(const DenseArgs& d, float* partial, cudaStream_t st);   // rows <= 32
int sa_module_simt(int b, int n, int m, int c, int nsample, const float* xyz, const float* new_xyz, const float* points,
                   const int* idx, const psa_mlp* mlp, float* out, cudaStream_t st);
int validate_mlp_public(const psa_mlp* mlp, const char* who);
int edgeconv_simt(int b, int n, int c, int k, const float* x, const int* nn_idx, const psa_mlp* mlp, float* out, cudaStream_t st);
// `run_if` non-null: no-op unless *run_if != 0 (device-side condition, see tc_mlp.cu)
int launch_fill_ord_neg_inf(long long total, float* out, cudaStream_t st, const unsigned int* run_if = nullptr);   // out := order-preserving int code of -inf
int launch_decode_ord(long long total, float* out, cudaStream_t st, const unsigned int* run_if = nullptr);         // int codes -> floats, in place
// edgeconv_train.cu: the backward of an EdgeConv layer that sees x (y_ij = Q_i + P_nn(i,j), PQ (b*n, 2N)) once its batch-norm coefficients
// coef (3, N) are known -> dW (2c, N), dx (b*n, c).  dz (b*n*k, N) gives the gradient w.r.t. the layer's batch-norm output per edge; when it
// is null, the max's gradient is routed by (pooled, R) as the single-layer op does.  dW null: dx only (frozen batch norm).
// workspace: edge_tail_workspace_bytes, 256-byte aligned.
size_t edge_tail_workspace_bytes(int b, int n, int c, int k, int N);
int edge_layer_tail(int b, int n, int c, int k, int N, const float* x, const int* nn_idx, const float* W, const float* PQ, const float* scale,
                    const float* shift, const float* coef, const float* pooled, const float* R, const float* dz, float* dW, float* dx,
                    void* workspace, cudaStream_t st);
// frozen batch norm's backward coefficients dy = scale * dz: coef (3, N) := (scale, 0, 0)
int frozen_coef(int N, const float* scale, float* coef, cudaStream_t st);

// tc_mlp.cu, shared with spider.cu: the arithmetic mode of psa_set_mlp_mode (0, 1, 2), the operand pieces of its tensor-core
// launches (2 or 3), the tile width (| format flag) of a dense layer, and the weight images (layout in tc_mlp.cu).
int mlp_mode();
int tc_np();
int tc_dense_nt(long long rows, int N);
// image of W (K x N, rows K..Kp zero) in the format `Nt` carries (width | format flag); `run_if` non-null: built only if *run_if != 0
int build_image(int K, int Kp, int N, int Nt, const float* W, uint8_t* image, cudaStream_t st, const unsigned int* run_if = nullptr);
const unsigned int* image_trailer(const uint8_t* image, int Kp, int N);   // fp16x2 image: the non-finite-weight word
const float* image_colscale(const uint8_t* image, int Kp, int N);         // fp16x2 image: the column factors 2^-e_n

}  // namespace psa

// tc_mlp.cu: W (2c, N) of a single-layer EdgeConv -> Wc (c, 2N) = [W_a - W_b | W_b] (grid-stride over the c * 2N entries)
__global__ void edge_wc_kernel(int c, int N, const float* __restrict__ W, float* __restrict__ Wc);
