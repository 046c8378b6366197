// ring_gemm.cu -- the launch of the shared ring GEMM (ring_gemm.cuh).
#include "ring_gemm.cuh"

namespace psa {

int ring_launch(const RingKernels& k, int np, int Nt, const void* args, long long units, cudaStream_t st) {
    const int nc = Nt / 64;
    const void* fn = k.fn[np - 2][nc - 1];
    const size_t smem = (size_t)ring_stages(np, nc, k.budget) * ring_stage_bytes(np, nc) + 1024;
    PSA_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int dev = 0, sms = 0;
    PSA_CUDA(cudaGetDevice(&dev));
    PSA_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    void* params[] = {const_cast<void*>(args)};
    cudaLaunchKernel(fn, dim3((unsigned)(units < sms ? units : sms)), dim3(kRingThreads), params, smem, st);   // its error is the last error
    return check_launch(k.name);
}

}  // namespace psa
