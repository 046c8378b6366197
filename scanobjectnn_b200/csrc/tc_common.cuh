// tc_common.cuh -- hand-written wgmma / TMA bulk copy / mbarrier wrappers for sm_90a (inline PTX, no CUTLASS).
//
// Conventions used by the kernels in tc_mlp.cu and knn_tc.cu:
//   * one WARPGROUP (4 warps, 128 threads) computes a 64-row tile: D[64 x 64] (+)= A[64 x 16] . B[16 x 64] per
//     wgmma.mma_async m64n64k16, fp32 accumulators in registers.  Warp w of the group holds rows 16w..16w+15; lane
//     (g = lane / 4, t = lane % 4) holds, of every 8-column block j, d[4j], d[4j+1] = row g, columns 8j+2t, 8j+2t+1 and
//     d[4j+2], d[4j+3] = the same columns of row g+8.  The A operand from registers has the matching layout (a0: row g,
//     k 2t..2t+1; a1: row g+8; a2, a3: k + 8), so the D of one layer becomes the A of the next without leaving registers;
//   * the B operand (weights, [N][K] "K-major") lives in shared memory in the canonical 128-byte-swizzle layout:
//     8-row x 128-byte atoms, 16-byte chunk index XOR (row % 8), atoms of consecutive 8-row groups 1024 B apart (SBO),
//     consecutive 128-byte K blocks N*128 B apart.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace psa {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// generic-proxy shared-memory writes -> visible to the async proxy (wgmma reads operands through descriptors)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }

// ---- mbarrier ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done;
    const uint32_t addr = smem_u32(bar);
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}\n"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
    } while (!done);
}
__device__ __forceinline__ void mbar_arrive1(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t warp_uniform(uint32_t v) { return __shfl_sync(0xffffffffu, v, 0); }
// named barrier `id` of `count` threads
__device__ __forceinline__ void unit_bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;\n" ::"r"(id), "r"(count) : "memory"); }

// ---- bulk async copy global -> shared (TMA engine, 1-D, no tensor map), completion on an mbarrier ----
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// ---- per-thread async copies global -> shared (cp.async); the thread's copies issued so far arrive on an mbarrier when done ----
__device__ __forceinline__ void cp_async16(uint32_t smem_dst, const void* gmem_src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(smem_dst), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t smem_dst, const void* gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(smem_dst), "l"(gmem_src) : "memory");
}
// counts as one of the barrier's expected arrivals (.noinc)
__device__ __forceinline__ void cp_async_mbar_arrive(uint64_t* bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}

// ---- descriptors ----
// wgmma shared-memory matrix descriptor, K-major, SWIZZLE_128B:
//   [0,14) start address >> 4 | [16,30) leading byte offset >> 4 (unused for swizzled K-major; 1) |
//   [32,46) stride byte offset >> 4 (1024 B between 8-row groups) | [62,64) layout type = 1 (128-byte swizzle)
// Moving the tile by `off` bytes (a multiple of 16 inside the 256 KB window, e.g. 32 B per 16-element K step) is one add on the
// start-address field.
__device__ __forceinline__ uint64_t wg_desc(uint32_t smem_addr) {
    const uint32_t lo = ((smem_addr & 0x3FFFFu) >> 4) | (1u << 16);
    const uint32_t hi = (1024u >> 4) | (1u << 30);
    return ((uint64_t)hi << 32) | lo;
}
constexpr uint32_t kFmtF16 = 0, kFmtBF16 = 1;

// ---- wgmma (whole warpgroup, converged) ----
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory"); }
// wait until at most N committed groups are pending (N = 1: the group committed last may still run)
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// accumulators are written asynchronously: after wg_wait_all, pin every read of them behind the wait
__device__ __forceinline__ void wg_fence_acc(float (&d)[32]) {
#pragma unroll
    for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 64] (+)= A[64 x 16] (registers, NP = 2: fp16, NP = 3: bf16) . B[16 x 64] (shared memory); accumulate = 0 overwrites D
template <int NP>
__device__ __forceinline__ void wg_mma_rs(float (&d)[32], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t bdesc, uint32_t accumulate) {
    if constexpr (NP == 2) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(bdesc), "r"(accumulate));
    } else {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(bdesc), "r"(accumulate));
    }
}
// D[64 x 64] (+)= A[64 x 16] . B[16 x 64], both bf16 from shared memory (K-major SWIZZLE_128B descriptors)
__device__ __forceinline__ void wg_mma_ss_bf16(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// ---- operand quantisation (done by us, so the tensor core only ever sees exactly representable values) ----
__device__ __forceinline__ float tf32_trunc(float x) { return __uint_as_float(__float_as_uint(x) & 0xffffe000u); }
__device__ __forceinline__ uint32_t pack_bf16x2(float lo_elem, float hi_elem) {
    __nv_bfloat162 p = __floats2bfloat162_rn(lo_elem, hi_elem);   // .x = lo_elem (low 16 bits), .y = hi_elem
    return *reinterpret_cast<uint32_t*>(&p);
}

// fp16 pieces (two per operand: 22 mantissa bits, three MMAs per product).  pack: .x = lo_elem in the low 16 bits.
__device__ __forceinline__ uint32_t pack_f16x2(float lo_elem, float hi_elem) {
    __half2 p = __floats2half2_rn(lo_elem, hi_elem);
    return *reinterpret_cast<uint32_t*>(&p);
}
__device__ __forceinline__ float2 unpack_f16x2(uint32_t p) { return __half22float2(*reinterpret_cast<__half2*>(&p)); }
// running |max| of every leading piece a kernel stores (packed halves): an infinity here means a value left the fp16 range
__device__ __forceinline__ void track_f16x2(uint32_t& m, uint32_t p) {
    const __half2 r = __hmax2(*reinterpret_cast<__half2*>(&m), __habs2(*reinterpret_cast<__half2*>(&p)));
    m = *reinterpret_cast<const uint32_t*>(&r);
}
__device__ __forceinline__ bool f16x2_overflowed(uint32_t m) { return (m & 0x7c00u) == 0x7c00u || (m & 0x7c000000u) == 0x7c000000u; }

// Operand split of the tensor-core kernels, NP pieces per operand:
//   NP = 3: three bf16 pieces (a = a1 + a2 + a3 exactly), six MMAs  a1w3 + a2w2 + a3w1 + a1w2 + a2w1 + a1w1  (small products first: the
//           accumulator add truncates) -- any fp32 magnitude;
//   NP = 2: two fp16 pieces (22 mantissa bits; the tail below 2^-24 absolute is dropped), three MMAs  a1w2 + a2w1 + a1w1 -- half
//           the tensor work, valid while |a| < 65504 (the kernels track the stored activation pieces and raise a flag otherwise;
//           the launcher then reruns the op on the NP = 3 instantiation).  Weights are split after a per-column power-of-two
//           scaling (tc_mlp.cu), so they keep 22 bits at any scale; activations keep an absolute 2^-25.
template <int NP> struct Split;
template <> struct Split<3> {
    static constexpr uint32_t kFmt = kFmtBF16;
    static constexpr int kTerms = 6;
    __host__ __device__ static constexpr uint32_t a(int t) { return t == 0 ? 0u : t == 1 ? 1u : t == 2 ? 2u : t == 3 ? 0u : t == 4 ? 1u : 0u; }
    __host__ __device__ static constexpr uint32_t w(int t) { return t == 0 ? 2u : t == 1 ? 1u : t == 2 ? 0u : t == 3 ? 1u : 0u; }
};
template <> struct Split<2> {
    static constexpr uint32_t kFmt = kFmtF16;
    static constexpr int kTerms = 3;
    __host__ __device__ static constexpr uint32_t a(int t) { return t == 1 ? 1u : 0u; }
    __host__ __device__ static constexpr uint32_t w(int t) { return t == 0 ? 1u : 0u; }
};
// split two consecutive elements into NP packed pieces p[0..NP) (h0, h1 are clobbered); NP = 2 also tracks the leading piece
template <int NP>
__device__ __forceinline__ void split_pair(float h0, float h1, uint32_t (&p)[NP], uint32_t& ovf) {
    if constexpr (NP == 3) {
        (void)ovf;
        p[0] = pack_bf16x2(h0, h1);
        h0 -= __uint_as_float(p[0] << 16); h1 -= __uint_as_float(p[0] & 0xffff0000u);
        p[1] = pack_bf16x2(h0, h1);
        h0 -= __uint_as_float(p[1] << 16); h1 -= __uint_as_float(p[1] & 0xffff0000u);
        p[2] = pack_bf16x2(h0, h1);
    } else {
        p[0] = pack_f16x2(h0, h1);
        track_f16x2(ovf, p[0]);
        const float2 f = unpack_f16x2(p[0]);
        p[1] = pack_f16x2(h0 - f.x, h1 - f.y);
    }
}

// ---- weight images (built by tc_mlp.cu's build_image; layout described there) ----
// np = pieces per weight: 3 (bf16x3, 6 bytes per weight) or 2 (fp16x2, 4 bytes); see Split<NP> above
__host__ __device__ constexpr uint32_t tc_block_bytes(int Nt, int np) { return (uint32_t)Nt * 128u * (uint32_t)np; }
__host__ __device__ inline size_t tc_image_bytes(int K, int N, int np) { return (size_t)K * N * 2u * (size_t)np; }     // independent of the tile width
// an image allocation = the blocks, np = 2: the N column factors 2^-e_n (fp32), then a 256-byte trailer whose first word is set
// when a weight is not finite (np = 2)
__host__ __device__ inline size_t tc_image_colscale_off(int K, int N, int np) { return (tc_image_bytes(K, N, np) + 255) & ~(size_t)255; }
__host__ __device__ inline size_t tc_image_trailer_off(int K, int N, int np) {
    return tc_image_colscale_off(K, N, np) + (np == 2 ? ((size_t)N * 4u + 255) & ~(size_t)255 : 0);
}
__host__ __device__ inline size_t tc_image_alloc_bytes(int K, int N, int np) { return tc_image_trailer_off(K, N, np) + 256; }

constexpr int kImageBf16x3 = 0x100;      // flags in psa_mlp.image_nt / psa_mlp_image_plan: image holds three bf16 pieces ..
constexpr int kImageF16x2 = 0x200;       // .. or two fp16 pieces
constexpr int kImageFlags = kImageBf16x3 | kImageF16x2;
__host__ __device__ inline int image_flag(int np) { return np == 2 ? kImageF16x2 : kImageBf16x3; }

// 1 / x, exactly, for a normal power of two x (the column factors): the exponent field mirrored about the bias, one integer
// subtraction instead of a correctly rounded reciprocal's slow path
__device__ __forceinline__ float pow2_rcp(float x) { return __int_as_float(0x7f000000 - __float_as_int(x)); }

// byte offset of element (n, k) of a [N][K] K-major SWIZZLE_128B tile
__device__ __forceinline__ uint32_t swz_off_f32(uint32_t n, uint32_t k, uint32_t N) {
    return (k >> 5) * (N * 128u) + (n >> 3) * 1024u + (n & 7u) * 128u + ((((k & 31u) >> 2) ^ (n & 7u)) << 4) + (k & 3u) * 4u;
}
__device__ __forceinline__ uint32_t swz_off_bf16(uint32_t n, uint32_t k, uint32_t N) {
    return (k >> 6) * (N * 128u) + (n >> 3) * 1024u + (n & 7u) * 128u + ((((k & 63u) >> 3) ^ (n & 7u)) << 4) + (k & 7u) * 2u;
}

}  // namespace tc
}  // namespace psa
