// Shared pieces of the self-attention kernels (attention.cu: whole head resident in shared memory, S <= 384;
// attention_stream.cu: K/V and Q/dO streamed through a shared-memory ring, any S): the XOR-swizzled [rows][64] bf16
// tile layout, its ldmatrix fragment loaders for mma.sync m16n8k16, cp.async with mbarrier completion, quad reductions.
#pragma once
#include "common.cuh"

namespace mmb {

constexpr int HD = 64;

// byte offset of element (r, c) (c multiple of 8) in a [rows][64] bf16 tile with 16B-chunk XOR swizzle
__device__ __forceinline__ uint32_t toff(int r, int c) { return (uint32_t)(r * 128 + ((((c >> 3) ^ (r & 7))) << 4)); }

// A fragment (16 rows x 16 k) at rows r0.., cols c0.. of a row-major tile
__device__ __forceinline__ void load_a(uint32_t (&a)[4], uint32_t base, int r0, int c0, int lane) {
  ldsm_x4(a, base + toff(r0 + (lane & 7) + ((lane >> 3) & 1) * 8, c0 + (lane >> 4) * 8));
}
// B fragments from a tile stored [n][k] (k contiguous): 8 n-rows at n0, 32 k at k0 -> {b0,b1} for k-step k0 and k0+16
__device__ __forceinline__ void load_b_nk(uint32_t (&b)[4], uint32_t base, int n0, int k0, int lane) {
  ldsm_x4(b, base + toff(n0 + (lane & 7), k0 + (lane >> 3) * 8));
}
// B fragments from a tile stored [k][n] (n contiguous): 16 k-rows at k0, 16 n at n0 -> {b0,b1} for n-tile n0 and n0+8
__device__ __forceinline__ void load_b_kn(uint32_t (&b)[4], uint32_t base, int k0, int n0, int lane) {
  ldsm_x4_t(b, base + toff(k0 + (lane & 7) + ((lane >> 3) & 1) * 8, n0 + (lane >> 4) * 8));
}

// 16-byte cp.async into shared memory; src_bytes = 0 writes zeros without reading src
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
// the mbarrier completes one arrival of this thread once all of its earlier cp.async copies have landed
__device__ __forceinline__ void cp_async_arrive(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// Streamed kernels (attention_stream.cu), used by attention.cu's entry points for S > 384.  Same arguments and
// output contract as the resident kernels; lse may be null in the forward.
int attention_fwd_stream(const void* qkv, void* out, float* lse, const uint8_t* kmask, int B, int S, int H, int causal,
                         float scale, cudaStream_t stream);
int attention_bwd_stream(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                         const uint8_t* kmask, int B, int S, int H, int causal, float scale, cudaStream_t stream);
constexpr int ATTN_BWD_STREAM_LAUNCHES = 2;   // dQ (and D) kernel, then the dK / dV kernel

}  // namespace mmb
