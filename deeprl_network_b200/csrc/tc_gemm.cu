// tc_gemm.cu -- weight packing for the tensor-core path + a stand-alone 3xTF32 GEMM used by the tests to
// validate the tensor-core pipeline (swizzled operand tiles, wgmma descriptors, bulk copies, mbarriers)
// in isolation:  C[M x N] = A[M x K] * W[K x N]   (M % 128 == 0, K % 8 == 0, N in {64, 128, 192, 256}).
#include "common.cuh"
#include "tc.cuh"

namespace {

// Packed operand: for every 32-wide k-block kb: [hi tile | lo tile], each tile = N rows x 128 B in the
// SWIZZLE_128B K-major layout (row n <-> output column n of W, i.e. the tile holds W^T).
__global__ void pack_b_kernel(const float* __restrict__ W, int ldw, int K, int n0, int nrows, float* __restrict__ out) {
  const int nkb = (K + 31) / 32;
  const int total = nkb * nrows * 32;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int n = idx % nrows;                 // consecutive threads -> consecutive columns of W (coalesced)
    const int kk = (idx / nrows) % 32;
    const int kb = idx / (nrows * 32);
    const int k = kb * 32 + kk;
    const float x = (k < K) ? W[(size_t)k * ldw + n0 + n] : 0.f;
    float hi, lo;
    tc::split_tf32(x, hi, lo);
    char* tile = reinterpret_cast<char*>(out) + (size_t)kb * 2 * nrows * 128;
    const uint32_t off = tc::sw128_offset(n, kk);
    *reinterpret_cast<float*>(tile + off) = hi;
    *reinterpret_cast<float*>(tile + (size_t)nrows * 128 + off) = lo;
  }
}

// 64 rows per CTA: warps 0-3 are the MMA warpgroup (accumulator in registers, written straight to C), warps 4-5
// produce the A operand (one row per thread) into the swizzled shared-memory ring, warp 6 bulk-copies B.
template <int N>
__global__ void __launch_bounds__(224, 1) tc_gemm_test_kernel(const float* __restrict__ A, int K, const float* __restrict__ Bp,
                                                              float* __restrict__ C, int* err) {
  constexpr int S = 2;                                   // B stages and A slots
  constexpr uint32_t TILE = N * 128;                     // bytes of one hi (or lo) B tile
  constexpr uint32_t STAGE = 2 * TILE;
  constexpr uint32_t A_TILE = 64 * 128, A_SLOT = 2 * A_TILE;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* bst = smem;
  uint8_t* ast = smem + S * STAGE;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ast + S * A_SLOT);
  uint64_t* b_full = bars, *b_empty = bars + S, *a_full = bars + 2 * S, *a_empty = bars + 3 * S;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nkb = (K + 31) / 32;
  if (tid == 0) {
    for (int s = 0; s < S; ++s) {
      tc::mbar_init(&b_full[s], 1); tc::mbar_init(&b_empty[s], 128);
      tc::mbar_init(&a_full[s], 64); tc::mbar_init(&a_empty[s], 128);
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    float d[N / 2];
#pragma unroll
    for (int j = 0; j < N / 2; ++j) d[j] = 0.f;
    for (int kb = 0; kb < nkb; ++kb) {
      const int st = kb % S;
      tc::mbar_wait(&b_full[st], (kb / S) & 1, err, 4);
      tc::mbar_wait(&a_full[st], (kb / S) & 1, err, 5);
      const int ksteps = min(4, (K - kb * 32) / 8);
      uint8_t* a = ast + st * A_SLOT;
      uint8_t* b = bst + st * STAGE;
      tc::wgmma_fence();
      tc::wgmma_kblock_3x(N, d, tc::smem_desc_sw128(a), tc::smem_desc_sw128(a + A_TILE), tc::smem_desc_sw128(b),
                          tc::smem_desc_sw128(b + TILE), ksteps, kb == 0);
      tc::wgmma_commit();
      tc::wgmma_wait_all();
      tc::mbar_arrive(&a_empty[st]);
      tc::mbar_arrive(&b_empty[st]);
    }
    const size_t r0 = (size_t)blockIdx.x * 64 + 16 * warp + (lane >> 2);
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
      const int col = 8 * j + 2 * (lane & 3);
      *reinterpret_cast<float2*>(C + r0 * N + col) = make_float2(d[4 * j], d[4 * j + 1]);
      *reinterpret_cast<float2*>(C + (r0 + 8) * N + col) = make_float2(d[4 * j + 2], d[4 * j + 3]);
    }
  } else if (warp < 6) {
    const int r = tid - 128;
    const size_t row = (size_t)blockIdx.x * 64 + r;
    for (int kb = 0; kb < nkb; ++kb) {
      const int st = kb % S;
      tc::mbar_wait(&a_empty[st], ((kb / S) & 1) ^ 1, err, 1);
      uint8_t* hi = ast + st * A_SLOT;
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        float x[8];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int k = kb * 32 + h * 8 + q * 4;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (k < K) v = *reinterpret_cast<const float4*>(A + row * K + k);
          x[4 * q] = v.x; x[4 * q + 1] = v.y; x[4 * q + 2] = v.z; x[4 * q + 3] = v.w;
        }
        tc::st_hilo8(hi, hi + A_TILE, (uint32_t)r, (uint32_t)(h * 8), x);
      }
      tc::fence_proxy_async();
      tc::mbar_arrive(&a_full[st]);
    }
  } else {
    if (lane == 0) {
      for (int kb = 0; kb < nkb; ++kb) {
        const int st = kb % S;
        tc::mbar_wait(&b_empty[st], ((kb / S) & 1) ^ 1, err, 3);
        tc::mbar_arrive_expect_tx(&b_full[st], STAGE);
        tc::bulk_g2s(bst + st * STAGE, reinterpret_cast<const uint8_t*>(Bp) + (size_t)kb * STAGE, STAGE, &b_full[st]);
      }
    }
  }
}

}  // namespace

int nmarl_launch_pack_b(const float* W, int ldw, int K, int n0, int nrows, float* out, cudaStream_t st) {
  const int total = ((K + 31) / 32) * nrows * 32;
  pack_b_kernel<<<(total + 255) / 256, 256, 0, st>>>(W, ldw, K, n0, nrows, out);
  NMARL_LAUNCH_CHECK();
  return 0;
}

// C[M x N] = A[M x K] * W[K x N]; scratch must hold ceil(K/32) * 2 * N * 32 floats; err: device int (0 = ok)
extern "C" __attribute__((visibility("default"))) int nmarl_tc_gemm_selftest(const float* A, const float* W, float* C, int M, int K,
                                                                               int N, float* scratch, int* err, void* stream) {
  NMARL_CHECK(M > 0 && M % 128 == 0 && K > 0 && K % 8 == 0 && (N == 64 || N == 128 || N == 192 || N == 256),
              "tc_gemm_selftest: unsupported shape");
  cudaStream_t st = (cudaStream_t)stream;
  if (nmarl_launch_pack_b(W, N, K, 0, N, scratch, st)) return 1;
  const size_t smem = 2 * 2 * (size_t)N * 128 + 2 * 2 * 64 * 128 + 1024 + 256;
  auto run = [&](auto kern) -> int {
    NMARL_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<M / 64, 224, smem, st>>>(A, K, scratch, C, err);
    NMARL_LAUNCH_CHECK();
    return 0;
  };
  switch (N) {     // one wgmma shape per width: m64n64k8, m64n128k8, m64n192k8, m64n256k8
    case 64: return run(tc_gemm_test_kernel<64>);
    case 128: return run(tc_gemm_test_kernel<128>);
    case 192: return run(tc_gemm_test_kernel<192>);
    default: return run(tc_gemm_test_kernel<256>);
  }
}
