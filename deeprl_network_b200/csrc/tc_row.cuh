// tc_row.cuh -- shared structure of the tensor-core cell kernels (forward: tc_cell.cu, backward: tc_bwd.cu):
// shared-memory map, k-block schedule entries, the row-thread producer helpers and the B-producer / MMA-warpgroup
// role loops.  See tc_cell.cu for the overall design.
#pragma once
#include "common.cuh"
#include "tc.cuh"

namespace tcrow {

constexpr int ROWS = 64;                                 // env rows of a CTA (= wgmma M)
constexpr int S_STAGES = 2;
constexpr uint32_t STAGE_BYTES = 2 * 256 * 128;          // hi+lo tiles of the widest operand (N = 256)
// A-operand ring in shared memory: A_SLOTS slots of [hi | lo] 64-row x 32-deep swizzled tiles
constexpr int A_SLOTS = 2;
constexpr uint32_t A_TILE = ROWS * 128, A_SLOT_BYTES = 2 * A_TILE;
static_assert((A_SLOTS & (A_SLOTS - 1)) == 0, "A ring slots: power of two");
// accumulator staging: [64 rows][256 columns] fp32; the MMA warpgroup stores finished GEMM results here and the row
// threads read them back by (row, column).  Columns are XOR-swizzled in 16-byte chunks by (row % 8) so that a warp
// (32 rows, same column) and the fragment stores both spread over all banks.
constexpr int ACC_COLS = 256;
constexpr uint32_t ACC_BYTES = ROWS * ACC_COLS * 4;
constexpr uint32_t ACC_COL = 0;
constexpr int MAX_KB = 24;
// NSET warp-sets share every env row: set s of row r works on columns [s*W, (s+1)*W) of each 32-wide input
// k-block and on hidden units [s*EW, (s+1)*EW) of the encoders / LSTM cell.
constexpr int NSET = 4;
constexpr int W = 32 / NSET, EW = 64 / NSET;
constexpr int ROW_WARPS = ROWS / 32;                      // warps per set
constexpr int ROW_THREADS = ROWS * NSET;
constexpr int MMA_WARP0 = ROW_THREADS / 32;               // warps [MMA_WARP0, +4): the MMA warpgroup
constexpr int TC_THREADS = ROW_THREADS + 128;
static_assert(MMA_WARP0 % 4 == 0, "the MMA warps must form an aligned warpgroup");
static_assert(W == 8 && EW % 8 == 0, "8-column operand pieces");

__device__ __forceinline__ uint32_t acc_idx(uint32_t row, uint32_t col) {
  return row * ACC_COLS + (col & ~31u) + ((((col >> 2) ^ row) & 7u) << 2) + (col & 3u);
}

constexpr int MAX_SEG = 8;
// The k-block schedule: a flat list of streamed weight k-blocks (thread 0 of the MMA warpgroup copies them in this
// order) and the GEMMs ("segments") it is made of.  A segment's width N is uniform over the CTA, so the MMA warpgroup
// dispatches on it once per GEMM and runs straight-line wgmma code of that width.
struct KbEnt { uint32_t off_bytes, bytes; };              // one [hi | lo] weight k-block in the packed operands
enum : uint8_t { DONE_NONE = 0, DONE_ENC, DONE_ACC };     // completion barrier a GEMM arrives on once stored
struct Seg {
  uint16_t n, dcol;                                       // GEMM width N, accumulator column of the result
  uint8_t kb0, nkb, ks_last, done;                        // k-blocks [kb0, kb0 + nkb), k-steps of the last one
};

struct RowCtx {
  uint8_t* a_ring; const float* acc;
  uint32_t r;                                             // env row of this thread inside the CTA
  uint64_t* a_full; uint64_t* a_empty; uint64_t* enc_full;
  int q, e, set;
  int* err;
};

__device__ __forceinline__ void produce_begin(RowCtx& c) {
  const int slot = c.q & (A_SLOTS - 1);
  tc::mbar_wait(&c.a_empty[slot], ((c.q / A_SLOTS) & 1) ^ 1, c.err, 11);
}
__device__ __forceinline__ void produce_piece(RowCtx& c, int col /*0..31, multiple of 8*/, const float (&x)[8]) {
  uint8_t* hi = c.a_ring + (c.q & (A_SLOTS - 1)) * A_SLOT_BYTES;
  tc::st_hilo8(hi, hi + A_TILE, c.r, (uint32_t)col, x);
}
__device__ __forceinline__ void produce_end(RowCtx& c) {
  tc::fence_proxy_async();
  tc::mbar_arrive(&c.a_full[c.q & (A_SLOTS - 1)]);
  c.q++;
}
// 8 accumulator columns [col, col + 8) of this thread's row
__device__ __forceinline__ void acc_ld8(const RowCtx& c, uint32_t col, float (&v)[8]) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float4 t = *reinterpret_cast<const float4*>(c.acc + acc_idx(c.r, col + 4 * h));
    v[4 * h] = t.x; v[4 * h + 1] = t.y; v[4 * h + 2] = t.z; v[4 * h + 3] = t.w;
  }
}
// one input k-block: this thread contributes columns [set*W, set*W + W)
__device__ __forceinline__ void produce_in(RowCtx& c, const float (&x)[W]) {
  produce_begin(c);
  produce_piece(c, c.set * W, x);
  produce_end(c);
}
// two k-blocks fed by a 64-wide activation vector of which this thread holds [set*EW, set*EW + EW)
__device__ __forceinline__ void produce_act(RowCtx& c, const float (&s)[EW]) {
#pragma unroll
  for (int hb = 0; hb < 2; ++hb) {
    produce_begin(c);
#pragma unroll
    for (int p = 0; p < EW / 8; ++p) {
      const int col = c.set * EW + 8 * p;
      if ((col >> 5) == hb) {
        float t[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) t[j] = s[8 * p + j];
        produce_piece(c, col & 31, t);
      }
    }
    produce_end(c);
  }
}
// wait for the encoder GEMMs issued so far
__device__ __forceinline__ void enc_wait(RowCtx& c) {
  tc::mbar_wait(c.enc_full, c.e & 1, c.err, 12);
  c.e++;
}
// this thread's EW columns of a 64-wide result block at accumulator column `col`
__device__ __forceinline__ void enc_load(RowCtx& c, uint32_t col, float (&v)[EW]) {
#pragma unroll
  for (int p = 0; p < EW / 8; ++p) {
    float t[8];
    acc_ld8(c, col + c.set * EW + 8 * p, t);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[8 * p + j] = t[j];
  }
}
// feature-major saved activations [feature][env]: lane == env row, so one warp access per feature is a single
// 128-byte line (the row-major form would touch 32 lines per access)
template <int NV>
__device__ __forceinline__ void st_fm(float* base, int f0, int B, int b, const float (&v)[NV], int n = NV) {
  // saved activations are written once and read once much later (BPTT): streaming stores keep them from
  // evicting the weights and the recurrent state the next calls re-read from L2.  Only the first n features are
  // stored: a section narrower than the thread's column slice must not spill into the next one.
#pragma unroll
  for (int j = 0; j < NV; ++j)
    if (j < n) __stcs(base + (size_t)(f0 + j) * B + b, v[j]);
}
template <int NV>
__device__ __forceinline__ void ld_fm(const float* base, int f0, int B, int b, float (&v)[NV]) {
#pragma unroll
  for (int j = 0; j < NV; ++j) v[j] = __ldcs(base + (size_t)(f0 + j) * B + b);
}
// state tensors (h, c, messages and their gradients): plane p of [planes][B][64] (env-major, FM = false) or
// [planes][64][B] (feature-major, FM = true: lane == env row -> one 128-byte line per warp access)
template <bool FM, int NV>
__device__ __forceinline__ void ld_state(const float* base, size_t plane, int b, int u0, int B, float (&v)[NV]) {
  if (FM) {
    const float* p = base + (plane * NH + u0) * (size_t)B + b;
#pragma unroll
    for (int j = 0; j < NV; ++j) v[j] = p[(size_t)j * B];
  } else {
    const float* p = base + (plane * (size_t)B + b) * NH + u0;
#pragma unroll
    for (int q = 0; q < NV / 4; ++q) {
      const float4 w = *reinterpret_cast<const float4*>(p + 4 * q);
      v[4 * q] = w.x; v[4 * q + 1] = w.y; v[4 * q + 2] = w.z; v[4 * q + 3] = w.w;
    }
  }
}
template <bool FM, int NV>
__device__ __forceinline__ void st_state(float* base, size_t plane, int b, int u0, int B, const float (&v)[NV]) {
  if (FM) {
    float* p = base + (plane * NH + u0) * (size_t)B + b;
#pragma unroll
    for (int j = 0; j < NV; ++j) p[(size_t)j * B] = v[j];
  } else {
    float* p = base + (plane * (size_t)B + b) * NH + u0;
#pragma unroll
    for (int q = 0; q < NV / 4; ++q) *reinterpret_cast<float4*>(p + 4 * q) = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
  }
}
template <int NV>
__device__ __forceinline__ void store_vec(float* dst, const float (&s)[NV]) {
#pragma unroll
  for (int q = 0; q < NV / 4; ++q) *reinterpret_cast<float4*>(dst + 4 * q) = make_float4(s[4 * q], s[4 * q + 1], s[4 * q + 2], s[4 * q + 3]);
}
__device__ __forceinline__ void bias_act(float (&v)[EW], const float* __restrict__ b, int act /*0 relu 1 tanh 2 none*/) {
#pragma unroll
  for (int q = 0; q < EW / 4; ++q) {
    const float4 bb = __ldg(reinterpret_cast<const float4*>(b) + q);
    const float z[4] = {v[4 * q] + bb.x, v[4 * q + 1] + bb.y, v[4 * q + 2] + bb.z, v[4 * q + 3] + bb.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) v[4 * q + j] = act == 0 ? fmaxf(z[j], 0.f) : (act == 1 ? tanhf(z[j]) : z[j]);
  }
}
// MUFU-based activations for the tensor-core epilogues (ex2.approx + rcp): absolute error ~1e-7, well inside the
// 1e-5 parity budget, ~6x fewer instructions than expf/tanhf + IEEE division.
__device__ __forceinline__ float frcp_(float x) {          // one MUFU.RCP (1 ulp), no IEEE fix-up path
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float fsigmoid(float x) { return frcp_(1.0f + __expf(-x)); }
__device__ __forceinline__ float ftanh(float x) { return fmaf(2.0f, frcp_(1.0f + __expf(-2.0f * x)), -1.0f); }
__device__ __forceinline__ void row_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(ROW_THREADS) : "memory"); }
__device__ __forceinline__ void mma_wg_sync() { asm volatile("bar.sync 2, 128;" ::: "memory"); }


// [B stages | A slots | accumulator staging | mbarriers | schedule], 1024-byte aligned tiles
struct Smem {
  uint8_t* bst; uint8_t* ast; float* acc;
  uint64_t *b_full, *a_full, *a_empty, *enc_full, *acc_full;
  int* n_kb; int* n_seg; KbEnt* sched; Seg* seg;
};

// Schedule builder (thread 0, before the roles start).  gemm() appends one GEMM D[64 x N] = A[64 x K] W[K x N] of
// the packed operand at float offset off: its ceil(K / 32) k-blocks in k order, or in the order `order` lists them.
// Only the last k-block may be partial, and only at N = 64 (K of the observation / fingerprint encoders); a GEMM
// without k-blocks (K = 0) adds nothing.
struct SchedBuilder {
  const Smem& s;
  int nk, ns;
  __device__ __forceinline__ explicit SchedBuilder(const Smem& sm) : s(sm), nk(0), ns(0) {}
  __device__ __forceinline__ void gemm(int off_floats, int N, int K, int dcol, uint8_t done, const int* order = nullptr) {
    const int nkb = (K + 31) / 32;
    if (nkb == 0) return;
    int kb = 0;
    for (int j = 0; j < nkb; ++j) {
      kb = order ? order[j] : j;
      s.sched[nk + j] = KbEnt{(uint32_t)(off_floats + kb * 2 * N * 32) * 4u, 2u * N * 128u};
    }
    const int k8 = (K + 7) / 8 * 8;
    s.seg[ns++] = Seg{(uint16_t)N, (uint16_t)dcol, (uint8_t)nk, (uint8_t)nkb, (uint8_t)min(4, (k8 - kb * 32) / 8), done};
    nk += nkb;
  }
  __device__ __forceinline__ void finish() { *s.n_kb = nk; *s.n_seg = ns; }
};

// ---- the MMA warpgroup ------------------------------------------------------------------------------------------
// All 128 threads run the GEMMs of the schedule in order; per 8-deep k-step the 3xTF32 wgmma chain hi*hi, hi*lo,
// lo*hi into the register accumulator.  Thread 0 also streams the weight k-blocks: one cp.async.bulk (TMA engine) per
// k-block into the S_STAGES ring.  One k-block of MMAs stays in flight: k-block q is issued before the warpgroup waits
// for q - 1 (wgmma.wait_group 1), and only then are q - 1's A slot (a_empty) and B stage (refilled with k-block
// q - 1 + S_STAGES) released.  At the end of a GEMM everything is retired, its last k-block released, and the result
// stored into the staging area at column dcol; then it arrives on its completion barrier.  a_empty / enc_full /
// acc_full count one arrival per thread.
struct MmaCtx {
  const Smem& s;
  const uint8_t* wp;
  int* err;
  int t, n_kb;
  __device__ __forceinline__ void fetch(int q) const {
    const int st = q % S_STAGES;
    const KbEnt e = s.sched[q];
    tc::mbar_arrive_expect_tx(&s.b_full[st], e.bytes);
    tc::bulk_g2s(s.bst + st * STAGE_BYTES, wp + e.off_bytes, e.bytes, &s.b_full[st]);
  }
  // k-block q has retired in every thread of the warpgroup: free its A slot and refill its B stage
  __device__ __forceinline__ void release(int q) const {
    tc::mbar_arrive(&s.a_empty[q & (A_SLOTS - 1)]);
    mma_wg_sync();
    if (t == 0 && q + S_STAGES < n_kb) fetch(q + S_STAGES);
  }
  // wait for k-block q's operands and issue its KS k-steps (one commit group)
  template <int N, int KS>
  __device__ __forceinline__ void issue(float* d, int q, bool first) const {
    const int st = q % S_STAGES, slot = q & (A_SLOTS - 1);
    tc::mbar_wait(&s.b_full[st], (q / S_STAGES) & 1, err, 31);
    tc::mbar_wait(&s.a_full[slot], (q / A_SLOTS) & 1, err, 32);
    const uint8_t* b = s.bst + st * STAGE_BYTES;
    const uint8_t* a = s.ast + slot * A_SLOT_BYTES;
    tc::wgmma_fence();
    tc::wgmma_kblock_3x<N, KS>(d, tc::smem_desc_sw128(a), tc::smem_desc_sw128(a + A_TILE), tc::smem_desc_sw128(b),
                               tc::smem_desc_sw128(b + N * 128), first);
    tc::wgmma_commit();
  }
};

// MMA loop options.  MMA_PIPE: keep one k-block in flight (above); without it every k-block is retired and released
// before the next is issued.  MMA_PARTIAL: the schedule has GEMMs whose last k-block is partial (the forward's
// observation / fingerprint encoders, N = 64); without it only whole k-blocks are compiled.
enum : int { MMA_PIPE = 1, MMA_PARTIAL = 2 };

template <int OPT, int N, int KS_LAST>
__device__ __forceinline__ void gemm_segment(const MmaCtx& x, const Seg& sg) {
  float d[N / 2];
#pragma unroll
  for (int j = 0; j < N / 2; ++j) d[j] = 0.f;
  const int q0 = sg.kb0, qe = q0 + sg.nkb - 1;             // qe: the (possibly partial) last k-block
  constexpr bool PIPE = (OPT & MMA_PIPE) != 0;
  for (int q = q0; q < qe; ++q) {
    x.issue<N, 4>(d, q, q == q0);
    if (!PIPE) { tc::wgmma_wait<0>(); x.release(q); }
    else if (q > q0) { tc::wgmma_wait<1>(); x.release(q - 1); }
  }
  x.issue<N, KS_LAST>(d, qe, qe == q0);
  tc::wgmma_wait<0>();
  if (PIPE && qe > q0) x.release(qe - 1);
  x.release(qe);
  const int w = x.t >> 5, l = x.t & 31;
  const uint32_t r0 = 16 * w + (l >> 2);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const uint32_t col = sg.dcol + 8 * j + 2 * (l & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h)
      *reinterpret_cast<float2*>(x.s.acc + acc_idx(r0 + 8 * h, col)) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
  }
}
// A partial last k-block occurs only in the N = 64 encoder GEMMs of the observations and fingerprints (K <= 32), so
// only N = 64 (with MMA_PARTIAL) has the shorter variants; false: the segment is not one this kernel can run.
template <int OPT, int N>
__device__ __forceinline__ bool gemm_segment_n(const MmaCtx& x, const Seg& sg) {
  if (sg.n != N) return false;
  if constexpr (N == 64 && (OPT & MMA_PARTIAL) != 0) {
    switch (sg.ks_last) {
      case 1: gemm_segment<OPT, N, 1>(x, sg); return true;
      case 2: gemm_segment<OPT, N, 2>(x, sg); return true;
      case 3: gemm_segment<OPT, N, 3>(x, sg); return true;
    }
  }
  if (sg.ks_last != 4) return false;
  gemm_segment<OPT, N, 4>(x, sg);
  return true;
}
// NS: the GEMM widths the kernel's schedule uses.  A segment no instantiation runs is a schedule bug: the warpgroup
// stops and reports tc_err 30 (the row threads' waits then time out instead of hanging).
template <int OPT, int... NS>
__device__ __forceinline__ void mma_loop(const Smem& s, const float* wpack, int* err) {
  const MmaCtx x{s, reinterpret_cast<const uint8_t*>(wpack), err, (int)threadIdx.x - MMA_WARP0 * 32, *s.n_kb};
  if (x.t == 0)
    for (int q = 0; q < S_STAGES && q < x.n_kb; ++q) x.fetch(q);
  const int n_seg = *s.n_seg;
  for (int i = 0; i < n_seg; ++i) {
    const Seg sg = s.seg[i];
    const bool known = (gemm_segment_n<OPT, NS>(x, sg) || ...);
    if (!known) { if (x.t == 0) atomicCAS(err, 0, 30); break; }
    if (sg.done == DONE_ENC) tc::mbar_arrive(s.enc_full);
    if (sg.done == DONE_ACC) tc::mbar_arrive(s.acc_full);
  }
}
__device__ __forceinline__ Smem smem_map(uint8_t* raw) {
  uint8_t* s = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~uintptr_t(1023));
  Smem m;
  m.bst = s;
  m.ast = s + S_STAGES * STAGE_BYTES;
  m.acc = reinterpret_cast<float*>(m.ast + A_SLOTS * A_SLOT_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(m.acc) + ACC_BYTES);
  m.b_full = bars; m.a_full = bars + S_STAGES; m.a_empty = m.a_full + A_SLOTS;
  m.enc_full = m.a_empty + A_SLOTS; m.acc_full = m.enc_full + 1;
  m.n_kb = reinterpret_cast<int*>(m.acc_full + 1);
  m.n_seg = m.n_kb + 1;
  m.sched = reinterpret_cast<KbEnt*>(m.n_kb + 2);
  m.seg = reinterpret_cast<Seg*>(m.sched + MAX_KB);
  return m;
}
__device__ __forceinline__ void init_barriers(const Smem& s) {
  for (int i = 0; i < S_STAGES; ++i) tc::mbar_init(&s.b_full[i], 1);
  for (int i = 0; i < A_SLOTS; ++i) { tc::mbar_init(&s.a_full[i], ROW_THREADS); tc::mbar_init(&s.a_empty[i], 128); }
  tc::mbar_init(s.enc_full, 128);
  tc::mbar_init(s.acc_full, 128);
  tc::fence_barrier_init();
}
constexpr size_t TC_SMEM = 1024 /*align slack*/ + S_STAGES * STAGE_BYTES + A_SLOTS * A_SLOT_BYTES + ACC_BYTES + 16 * 8 /*mbarriers*/ +
                           8 + MAX_KB * sizeof(KbEnt) + MAX_SEG * sizeof(Seg);
static_assert(TC_SMEM <= 232448, "cell kernels exceed the 227 KB of dynamic shared memory");

}  // namespace tcrow
