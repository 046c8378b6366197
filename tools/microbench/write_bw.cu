// write_bw.cu -- ceiling for a pure write stream on H100 (what the F1 kernel's 134 MB output can reach at best).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o write_bw write_bw.cu && ./write_bw
// Variants: per-lane st.global.cs.v4 (streaming), plain st.global.v4, cp.async.bulk shared->global (16 KB chunks).
// Each is timed (a) isolated: 256 MB read-flush of L2 in front (clean lines), one launch; (b) steady state: 20 launches
// back to back into the same buffer (every byte has to reach HBM).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

template <int MODE>
__global__ void __launch_bounds__(256) st_kernel(float4* __restrict__ out, size_t n4) {
    // CTA owns a contiguous range; a warp instruction writes 512 contiguous bytes
    const size_t per = (n4 + gridDim.x - 1) / gridDim.x;
    const size_t lo = per * blockIdx.x, hi = lo + per < n4 ? lo + per : n4;
    const float4 v = make_float4(1.f, 2.f, 3.f, (float)threadIdx.x);
    for (size_t i = lo + threadIdx.x; i < hi; i += 256) {
        if (MODE == 0) __stcs(out + i, v);
        else out[i] = v;
    }
}

__global__ void __launch_bounds__(128) bulk_kernel(float4* __restrict__ out, size_t n4) {
    extern __shared__ __align__(128) float4 tile[];   // 16 KB
    constexpr int CH = 1024;                            // float4 per chunk = 16 KB
    for (int i = threadIdx.x; i < CH; i += 128) tile[i] = make_float4(1.f, 2.f, 3.f, (float)i);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const size_t nch = n4 / CH;
    if (threadIdx.x == 0) {
        const uint32_t src = (uint32_t)__cvta_generic_to_shared(tile);
        for (size_t c = blockIdx.x; c < nch; c += gridDim.x) {
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(out + c * CH), "r"(src), "r"(CH * 16) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            asm volatile("cp.async.bulk.wait_group.read 4;" ::: "memory");
        }
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

__global__ void read_flush(const float4* __restrict__ p, size_t n4, float* sink) {
    float acc = 0.f;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) acc += __ldcg(p + i).x;
    if (acc == 12345.678f) *sink = acc;
}

int main() {
    const size_t bytes = 134217728 + 2097152 + 65536;   // the F1 output of SA1: pre + idx + pts_cnt
    const size_t n4 = bytes / 16;
    float4 *out, *flush; float* sink;
    CK(cudaMalloc(&out, bytes)); CK(cudaMalloc(&flush, (size_t)256 << 20)); CK(cudaMalloc(&sink, 4));
    CK(cudaMemset(flush, 0, (size_t)256 << 20));
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    CK(cudaFuncSetAttribute(bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384));
    const int grids[3] = {148, 296, 592};
    for (int mode = 0; mode < 3; ++mode) {
        for (int gi = 0; gi < 3; ++gi) {
            const int g = grids[gi];
            auto launch = [&]() {
                if (mode == 0) st_kernel<0><<<g, 256>>>(out, n4);
                else if (mode == 1) st_kernel<1><<<g, 256>>>(out, n4);
                else bulk_kernel<<<g, 128, 16384>>>(out, n4);
            };
            for (int w = 0; w < 3; ++w) launch();
            CK(cudaDeviceSynchronize());
            float best = 1e9f, med[9];
            for (int r = 0; r < 9; ++r) {
                read_flush<<<592, 256>>>(flush, ((size_t)256 << 20) / 16, sink);
                CK(cudaEventRecord(e0)); launch(); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
                float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); med[r] = ms; if (ms < best) best = ms;
            }
            for (int i = 0; i < 9; ++i) for (int j = i + 1; j < 9; ++j) if (med[j] < med[i]) { float t = med[i]; med[i] = med[j]; med[j] = t; }
            CK(cudaEventRecord(e0));
            for (int r = 0; r < 20; ++r) launch();
            CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
            float ms20; CK(cudaEventElapsedTime(&ms20, e0, e1));
            printf("{\"mode\": \"%s\", \"ctas\": %d, \"bytes\": %zu, \"isolated_us_median\": %.2f, \"isolated_us_best\": %.2f, \"isolated_gbs\": %.0f, "
                   "\"steady_us\": %.2f, \"steady_gbs\": %.0f}\n",
                   mode == 0 ? "st.global.cs.v4" : (mode == 1 ? "st.global.v4" : "cp.async.bulk 16KB"), g, bytes, med[4] * 1e3, best * 1e3,
                   bytes / (med[4] * 1e-3) / 1e9, ms20 / 20 * 1e3, bytes / (ms20 / 20 * 1e-3) / 1e9);
        }
    }
    return 0;
}
