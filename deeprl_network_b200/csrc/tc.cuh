// tc.cuh -- Hopper (sm_90a) tensor-core primitives used by the 3xTF32 GEMMs:
// wgmma.mma_async kind tf32 with both operands in 128B-swizzled shared memory (the weight operand staged by
// cp.async.bulk + mbarrier, the activation operand written by the CUDA cores), FP32 accumulators in the registers of
// the issuing warpgroup.  Inline PTX only (no CUTLASS dependency).
//
// fp32-accurate products on TF32 tensor cores ("3xTF32"): x = hi + lo with hi = x ROUNDED to TF32
// (cvt.rna.tf32) and lo = the remainder x - hi (exact in fp32) rounded to TF32 as well.
// a*b ~= a_hi*b_hi + a_hi*b_lo + a_lo*b_hi; the dropped terms are O(2^-22 |a||b|) and -- because both parts are
// rounded to nearest -- zero-mean.  (The cheaper split, hi = x & 0xFFFFE000 with the hardware truncating lo, makes
// hi, lo and the dropped lo*lo term all err toward zero: a systematic ~2e-7 relative bias per product that does not
// average out over long contractions and is amplified by cancellation.)  Accumulation is FP32.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace tc {

// TF32 rounding / 3xTF32 operand split (see the header comment)
__device__ __forceinline__ uint32_t tf32_rn(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = tf32_rn(x);
  lo = tf32_rn(x - __uint_as_float(hi));
}
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  uint32_t h, l;
  split_tf32(x, h, l);
  hi = __uint_as_float(h); lo = __uint_as_float(l);
}
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- programmatic dependent launch (PDL) --------------------------------------------------------------------
// A kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may start while its predecessor in the
// stream is still running; it must execute pdl_wait() before touching anything the predecessor wrote (the wait returns
// once the predecessor grid has completed and its writes are visible).  pdl_launch_dependents() lets the NEXT
// kernel's CTAs be scheduled onto free SMs as soon as every CTA of this grid has started.  Both are no-ops for a
// kernel launched without the attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// One elected lane of a converged warp (the bulk-copy producer).  ptxas treats a branch on elect.sync as
// single-threaded, so the copy operands stay in uniform registers.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier ---------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// Bounded wait: a protocol bug must not hang the GPU.  The deadline is in SM clock cycles (~70 ms); once any
// wait of the grid has timed out (*err != 0) every later wait gives up immediately so the kernel drains.
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity, int* err, int code) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done = 0;
  long long t0 = 0;
  for (uint32_t spins = 0;; ++spins) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (done) return true;
    // The watchdog (clock + the grid-wide abort flag in global memory) is consulted only every 64th failed try_wait:
    // a global load per poll keeps the thread away from the barrier for an L2 round trip (~700 cycles) and that
    // latency was added to every wake-up of every fine-grained pipeline wait.
    if ((spins & 63u) != 63u) continue;
    const long long now = clock64();
    if (t0 == 0) t0 = now;
    if (now - t0 > (1ll << 27)) break;
    if (err != nullptr && *reinterpret_cast<volatile int*>(err) != 0) return false;
  }
  if (err != nullptr) atomicCAS(err, 0, code);
  return false;
}

// ---- bulk async copy global -> shared (TMA engine, 1-D) -------------------------------------------------
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---- shared-memory operand tiles + warpgroup MMA (wgmma) -------------------------------------------------------
// K-major operand tile [rows][32 tf32] in SWIZZLE_128B layout: row r at (r/8)*1024 + (r%8)*128 bytes, the
// eight 16-byte chunks of a row XOR-ed with (r%8).  Tiles start on a 1024-byte boundary.
__host__ __device__ inline uint32_t sw128_offset(uint32_t row, uint32_t k) {
  return (row >> 3) * 1024u + (row & 7u) * 128u + ((((k >> 2) ^ row) & 7u) << 4) + ((k & 3u) << 2);
}
// wgmma shared-memory descriptor of such a tile: start address >> 4, LBO unused (16 B), SBO = 1024 B between
// 8-row groups, layout type 1 = SWIZZLE_128B.  Advancing the start address by 32 B (+2) selects the next 8-deep k-step.
__device__ __forceinline__ uint64_t smem_desc_sw128(const void* tile) {
  const uint64_t addr = (uint64_t)(smem_u32(tile) >> 4) & 0x3FFFull;
  return addr | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
// 8 consecutive k of one row: hi tile and lo tile (3xTF32 split of x)
__device__ __forceinline__ void st_hilo8(uint8_t* tile_hi, uint8_t* tile_lo, uint32_t row, uint32_t k0, const float (&x)[8]) {
  float h[8], l[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) split_tf32(x[i], h[i], l[i]);
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const uint32_t off = sw128_offset(row, k0 + 4 * c);
    *reinterpret_cast<float4*>(tile_hi + off) = make_float4(h[4 * c], h[4 * c + 1], h[4 * c + 2], h[4 * c + 3]);
    *reinterpret_cast<float4*>(tile_lo + off) = make_float4(l[4 * c], l[4 * c + 1], l[4 * c + 2], l[4 * c + 3]);
  }
}
// operand tiles written with ordinary st.shared must be made visible to the async proxy (tensor core reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// wait until at most N committed wgmma groups of this warp are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x N] (+)= A[64 rows x 8 tf32, smem desc] * B[N rows x 8 tf32, smem desc]^T, issued by one whole warpgroup.
// Accumulator fragment (N/2 floats per thread): d[4j + {0,1}] = row 16*warp + lane/4, columns 8j + 2*(lane%4) + {0,1};
// d[4j + {2,3}] = the same columns of row + 8.
__device__ __forceinline__ void wgmma_tf32_n64(float* d, uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n128(float* d, uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n192(float* d, uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %98, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n192k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95}, %96, %97, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
      : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n256(float* d, uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32(int N, float* d, uint64_t da, uint64_t db, uint32_t acc) {
  switch (N) {
    case 64: wgmma_tf32_n64(d, da, db, acc); break;
    case 128: wgmma_tf32_n128(d, da, db, acc); break;
    case 192: wgmma_tf32_n192(d, da, db, acc); break;
    default: wgmma_tf32_n256(d, da, db, acc); break;
  }
}
template <int N>
__device__ __forceinline__ void wgmma_tf32(float* d, uint64_t da, uint64_t db, uint32_t acc) {
  static_assert(N == 64 || N == 128 || N == 192 || N == 256, "wgmma tf32 widths used here");
  if constexpr (N == 64) wgmma_tf32_n64(d, da, db, acc);
  else if constexpr (N == 128) wgmma_tf32_n128(d, da, db, acc);
  else if constexpr (N == 192) wgmma_tf32_n192(d, da, db, acc);
  else wgmma_tf32_n256(d, da, db, acc);
}
// the first KS 8-deep k-steps of a 32-deep k-block of a 3xTF32 GEMM of width N, straight-line code
template <int N, int KS>
__device__ __forceinline__ void wgmma_kblock_3x(float* d, uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo, bool first) {
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) {
    wgmma_tf32<N>(d, a_hi + 2 * ks, b_hi + 2 * ks, (first && ks == 0) ? 0u : 1u);
    wgmma_tf32<N>(d, a_hi + 2 * ks, b_lo + 2 * ks, 1u);
    wgmma_tf32<N>(d, a_lo + 2 * ks, b_hi + 2 * ks, 1u);
  }
}
// one 32-deep k-block of a 3xTF32 GEMM: a_hi*b_hi + a_hi*b_lo + a_lo*b_hi per 8-deep k-step
__device__ __forceinline__ void wgmma_kblock_3x(int N, float* d, uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo,
                                                int ksteps, bool first) {
  for (int ks = 0; ks < ksteps; ++ks) {
    wgmma_tf32(N, d, a_hi + 2 * ks, b_hi + 2 * ks, (first && ks == 0) ? 0u : 1u);
    wgmma_tf32(N, d, a_hi + 2 * ks, b_lo + 2 * ks, 1u);
    wgmma_tf32(N, d, a_lo + 2 * ks, b_hi + 2 * ks, 1u);
  }
}

}  // namespace tc
