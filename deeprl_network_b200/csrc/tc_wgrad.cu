// tc_wgrad.cu -- tensor-core (wgmma) weight gradients of every GEMM of the cell (gate matrix and the obs /
// fingerprint / message encoders):   dW[ka][n] = sum over all (t, env) rows r of  A[r][ka] * D[r][n]
// as 3xTF32 GEMMs with M = ka (one CTA per 128-lane job tile: two MMA warpgroups of 64 lanes each share every
// streamed D^T tile), the contraction over rows split across CTAs and a fixed-order reduce afterwards.
//   A operand: the saved activations are feature-major ([t][agent][feature][env]); operand row = feature ka, so
//              a thread reads the 32 consecutive envs of one k-block (one 128-byte line), splits hi/lo and stores
//              them into the swizzled shared-memory ring.
//   B operand: D^T, K-major over rows, was written by the backward cell kernel as raw fp32 128B-swizzled tiles
//              (dz: 256 rows, encoder pre-activation grads: 192/128/64 rows; nmarl_tc_tile_offset); one thread
//              bulk-copies the needed row range of the tile per 32 env rows and the A producers split it into
//              [hi | lo] in shared memory.
//   Biases:    the obs-encoder job carries an extra all-ones lane and spans every column of the dpre tile, which
//              yields all encoder bias gradients for free; the gate bias is a coalesced column sum of dz.
#include "bwd_common.cuh"
#include "tc_row.cuh"

extern long long* g_nmarl_prof;          // api.cu: debug hook (nmarl_debug_set_prof)

namespace {
using namespace tcrow;

enum { J_GATE0 = 0, J_GATE1, J_ENC_X, J_ENC_M0, J_ENC_M1, J_COUNT };
// Warpgroup 0: the A producers, one thread per feature lane of the 128-lane tile.  Warpgroups 1 and 2: the MMA
// warpgroups of lanes 0-63 and 64-127.
constexpr int WG_LANES = 128, WG_HALF = 64;
constexpr int WG_A_THREADS = WG_LANES, WG_THREADS = WG_A_THREADS + 2 * 128;
// A slot: [hi | lo] 128-row x 32-deep swizzled tiles; rows 64-127 of each form a second 1024-aligned 8 KB tile
constexpr uint32_t WG_A_TILE = WG_LANES * 128, WG_A_SLOT = 2 * WG_A_TILE;
// The B stages ([hi | lo] N-row tiles, 256 N bytes) and the A slots share one 224 KB ring; the depths depend on the
// job's N (wg_depths), so the narrow jobs run a much deeper ring than the gate jobs.
constexpr uint32_t WG_RING = 224 * 1024;
constexpr int WG_MAX_BARS = 32;
constexpr size_t WG_SMEM = 1024 + WG_RING + WG_MAX_BARS * 8;
static_assert(WG_SMEM <= 232448, "wgrad rings exceed the 227 KB of dynamic shared memory");
static_assert(WG_HALF == ROWS, "each MMA warpgroup covers the 64 rows of one wgmma");
// Register split (setmaxnreg): the CTA is launched with 168 registers per thread (384 x 168 = 64 512); the producer
// warpgroup drops to 120 and each MMA warpgroup (128 accumulators) rises to 192: 128 x 120 + 256 x 192 = 64 512.
constexpr int WG_REGS_A = 120, WG_REGS_MMA = 192;
static_assert(WG_A_THREADS * WG_REGS_A + 256 * WG_REGS_MMA <= WG_THREADS * 168, "setmaxnreg split exceeds the CTA's registers");
constexpr int SEG_KB = 20;       // k-blocks (of 32 rows) accumulated in registers before the accumulator is drained

// B stages and A slots per job width: N = 256: 2 x 64 KB + 3 x 32 KB; N = 192: 3 x 48 KB + 2 x 32 KB;
// N = 128: 4 x 32 KB + 3 x 32 KB; N = 64: 6 x 16 KB + 4 x 32 KB (DESIGN 4.1)
__device__ __forceinline__ void wg_depths(int N, int& S, int& A) {
  S = N >= 256 ? 2 : (N >= 192 ? 3 : (N >= 128 ? 4 : 6));
  A = (int)((WG_RING - (uint32_t)S * 256u * (uint32_t)N) / WG_A_SLOT);
  if (A > 4) A = 4;
}

// position in a ring of `n` entries: index and the parity of its current use
struct RingPos {
  int idx = 0; uint32_t ph = 0;
  __device__ __forceinline__ void next(int n) { if (++idx == n) { idx = 0; ph ^= 1u; } }
};

struct TcWgK {
  int B, T, splits, ndp;
  const float* sv_sh; const float* sv_xin; const float* dzT; const float* dpT;
  const float* h_seq; const float* done_pre;   // all but DIAL (feature-major state): h^ / m~ operand rows come from h_seq
  float* ws;
  long long ws_off[J_COUNT];     // float offset of each job's partial block [splits][N_agents][128][N_job]
  int jobs[J_COUNT]; int n_jobs; // job kinds present
  int* err;
  long long* prof;               // debug: per-k-block clock64 stamps of CTA (split 0, agent 0) of every job, or NULL
};

struct JobDesc {
  const float* A; int F_A, a_feat0, ka_cnt, ones;
  int p_feat0, p_cnt;             // obs-encoder job only: fingerprint features ride on the lanes behind the ones lane
  const float* BT; int tile_rows, n_row0, N;
};

__device__ __forceinline__ JobDesc job_desc(const nmarl_model& m, const TcWgK& k, int kind, int i) {
  const nmarl_agent& ag = m.agent[i];
  JobDesc d;
  d.p_feat0 = 0; d.p_cnt = 0;
  const int SD = m.s_dim, LDI = m.kx_pad + m.kp_pad + m.km_pad;
  const int Km = (m.variant == NMARL_IC3) ? NH : ag.n_nbr * NH;
  if (kind == J_GATE0 || kind == J_GATE1) {
    const int mt = kind - J_GATE0;
    d.A = k.sv_sh; d.F_A = SD + NH; d.a_feat0 = 128 * mt; d.ka_cnt = max(0, min(128, SD + NH - 128 * mt)); d.ones = 0;
    d.BT = k.dzT; d.tile_rows = 256; d.n_row0 = 0; d.N = 256;
  } else if (kind == J_ENC_X) {
    d.A = k.sv_xin; d.F_A = LDI; d.a_feat0 = 0; d.ka_cnt = ag.x_nsrc * ag.x_w; d.ones = 1;
    if (m.variant == NMARL_NC) { d.p_feat0 = m.kx_pad; d.p_cnt = ag.n_nbr * m.n_a; }
    d.BT = k.dpT; d.tile_rows = k.ndp; d.n_row0 = 0; d.N = k.ndp;
  } else {
    const int mt = kind - J_ENC_M0;
    d.A = k.sv_xin; d.F_A = LDI; d.a_feat0 = m.kx_pad + m.kp_pad + 128 * mt; d.ka_cnt = max(0, min(128, Km - 128 * mt)); d.ones = 0;
    d.BT = k.dpT; d.tile_rows = k.ndp; d.n_row0 = (m.variant == NMARL_NC) ? 128 : 64; d.N = 64;
  }
  return d;
}

// The D^T tiles hold raw fp32.  One tile per k-block is copied into the hi half of the stage; the A-producer threads
// split it in place into its rounded [hi | lo] pair (tc::split_tf32) and signal b_split, so the split overlaps the
// previous k-block's MMAs instead of preceding the k-block's own.
//
// Hand-offs per k-block q (B stage st = q mod S, A slot = q mod A; every wait is on an mbarrier):
//   thread 0 of MMA warpgroup 0 bulk-copies tile q into st once b_empty[st] reports that every active warpgroup has
//   retired k-block q - S;  the producers fill the A slot once a_empty reports the same for q - A, then split
//   stage st once b_full[st] has landed;  each active MMA warpgroup waits for b_split and a_full, issues its
//   12 wgmma against its own 64 A rows and the shared B stage, retires them and arrives on a_empty and b_empty (one
//   arrival per warp, so both count 4 x the active warpgroups).
// A warpgroup whose 64 lanes all lie beyond the job's real lanes (ka_cnt + ones lane + fingerprints) issues nothing:
// the reduce never reads those lanes.
__global__ void __launch_bounds__(WG_THREADS, 1) tc_wgrad_kernel(const __grid_constant__ nmarl_model m,
                                                                 const __grid_constant__ TcWgK k) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  const int sp = blockIdx.x, jslot = blockIdx.y, i = blockIdx.z;
  const int kind = k.jobs[jslot];
  const JobDesc d = job_desc(m, k, kind, i);
  const int lanes = d.ka_cnt > 0 ? d.ka_cnt + d.ones + d.p_cnt : 0;  // lanes the reduce reads (all zero if no features)
  const int nact = (lanes + WG_HALF - 1) / WG_HALF;                   // active MMA warpgroups: 0, 1 or 2
  if (nact == 0) return;                                              // nothing is read from this CTA's block
  int S, AS;
  wg_depths(d.N, S, AS);
  uint8_t* bst = smem;
  uint8_t* ast = smem + (size_t)S * 256 * d.N;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + WG_RING);
  uint64_t *b_full = bars, *b_split = b_full + S, *b_empty = b_split + S, *a_full = b_empty + S, *a_empty = a_full + AS;

  const int N_agents = m.n_agent;
  const int tid = threadIdx.x, warp = tid >> 5;
  const int bpt = k.B / 32;                                           // 32-row k-blocks per time step
  const int kb_total = k.T * bpt;
  const int per = (kb_total + k.splits - 1) / k.splits;
  const int kb0 = sp * per, kb1 = min(kb_total, kb0 + per);
  const int nkb = (d.ka_cnt > 0) ? max(0, kb1 - kb0) : 0;
  float* wsj = k.ws + k.ws_off[jslot] + ((size_t)sp * N_agents + i) * 128 * d.N;

  if (tid == 0) {
    for (int s = 0; s < S; ++s) { tc::mbar_init(&b_full[s], 1); tc::mbar_init(&b_split[s], WG_A_THREADS); tc::mbar_init(&b_empty[s], 4 * nact); }
    for (int s = 0; s < AS; ++s) { tc::mbar_init(&a_full[s], WG_A_THREADS); tc::mbar_init(&a_empty[s], 4 * nact); }
    tc::fence_barrier_init();
  }
  __syncthreads();
  const uint32_t tile_bytes = (uint32_t)d.N * 128u;                   // hi (or lo) part staged per k-block

  if (warp < WG_A_THREADS / 32) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(WG_REGS_A));
    // ---- A producers: feature lane `row` of the job's 128-lane tile, all 32 envs of every k-block ----------------
    const int row = tid;
    const bool on = row < WG_HALF * nact;                             // an active warpgroup reads this row
    const int ka = row;
    const bool one = d.ones && ka == d.ka_cnt;
    const bool is_p = ka > d.ka_cnt && ka <= d.ka_cnt + d.p_cnt;
    const bool real = on && (ka < d.ka_cnt || is_p);
    const int feat = is_p ? d.p_feat0 + (ka - d.ka_cnt - 1) : d.a_feat0 + ka;
    // Feature-major state (all but DIAL): the forward kernel does not save h^ (= (1 - done) * own h_seq[t]) and, for
    // NeurComm, m~ (= the neighbours' h_seq[t]) a second time; those operand rows are read from the state sequence.
    int hs_agent = -1, hs_unit = 0;
    bool hs_mask = false;
    if (k.h_seq != nullptr && real && !is_p) {
      if ((kind == J_GATE0 || kind == J_GATE1) && feat >= m.s_dim) { hs_agent = i; hs_unit = feat - m.s_dim; hs_mask = true; }
      else if ((kind == J_ENC_M0 || kind == J_ENC_M1) && m.variant == NMARL_NC) {
        const int fm = feat - (m.kx_pad + m.kp_pad);
        hs_agent = m.agent[i].nbr[fm / NH]; hs_unit = fm % NH;
      }
    }
    // the A operand of k-block q: the 32 envs of this thread's feature (global loads; issued two k-blocks AHEAD so
    // that their latency hides behind the barrier waits of the current k-block)
    auto load_x = [&](int q, float (&x)[32]) {
      const int kb = kb0 + q, t = kb / bpt, rb = kb - t * bpt;
      if (hs_agent >= 0) {
        const float* src = k.h_seq + (((size_t)t * N_agents + hs_agent) * NH + hs_unit) * k.B + rb * 32;
#pragma unroll
        for (int p = 0; p < 8; ++p) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(src + 4 * p));
          x[4 * p] = v.x; x[4 * p + 1] = v.y; x[4 * p + 2] = v.z; x[4 * p + 3] = v.w;
        }
        if (hs_mask) {
          const float* dn = k.done_pre + (size_t)t * k.B + rb * 32;
#pragma unroll
          for (int p = 0; p < 8; ++p) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(dn + 4 * p));
            x[4 * p] *= 1.0f - v.x; x[4 * p + 1] *= 1.0f - v.y; x[4 * p + 2] *= 1.0f - v.z; x[4 * p + 3] *= 1.0f - v.w;
          }
        }
      } else if (real) {
        const float* src = d.A + (((size_t)t * N_agents + i) * d.F_A + feat) * k.B + rb * 32;
#pragma unroll
        for (int p = 0; p < 8; ++p) {
          const float4 v = __ldcs(reinterpret_cast<const float4*>(src + 4 * p));
          x[4 * p] = v.x; x[4 * p + 1] = v.y; x[4 * p + 2] = v.z; x[4 * p + 3] = v.w;
        }
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j) x[j] = one ? 1.0f : 0.0f;
      }
    };
    float xa[32], xb[32];                     // the operands of the next two k-blocks (two loads in flight per thread)
    RingPos as, bs;
    auto emit_a = [&](int q, float (&x)[32]) {
      tc::mbar_wait(&a_empty[as.idx], as.ph ^ 1, k.err, 11);
      if (on) {
        uint8_t* hi = ast + (size_t)as.idx * WG_A_SLOT;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          float x8[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) x8[j] = x[8 * c + j];
          tc::st_hilo8(hi, hi + WG_A_TILE, (uint32_t)row, (uint32_t)(8 * c), x8);
        }
        tc::fence_proxy_async();
      }
      tc::mbar_arrive(&a_full[as.idx]);
      as.next(AS);
      if (q + 2 < nkb) load_x(q + 2, x);        // refill this buffer; it is consumed two k-blocks from now
      // split the raw D^T tile of this k-block into its [hi | lo] pair once it has landed.  In order: the stage is
      // refilled with k-block q + S only after the MMAs of q, which wait for this split, have retired.
      tc::mbar_wait(&b_full[bs.idx], bs.ph, k.err, 31);
      float4* bhi = reinterpret_cast<float4*>(bst + (size_t)bs.idx * 2 * tile_bytes);
      float4* blo = reinterpret_cast<float4*>(bst + (size_t)bs.idx * 2 * tile_bytes + tile_bytes);
      for (uint32_t e = (uint32_t)tid; e < tile_bytes / 16; e += WG_A_THREADS) {
        const float4 v = bhi[e];
        float4 h, lo4;
        tc::split_tf32(v.x, h.x, lo4.x); tc::split_tf32(v.y, h.y, lo4.y);
        tc::split_tf32(v.z, h.z, lo4.z); tc::split_tf32(v.w, h.w, lo4.w);
        bhi[e] = h;
        blo[e] = lo4;
      }
      tc::fence_proxy_async();
      tc::mbar_arrive(&b_split[bs.idx]);
      bs.next(S);
    };
    if (nkb > 0) load_x(0, xa);
    if (nkb > 1) load_x(1, xb);
    for (int q = 0; q < nkb; q += 2) {
      emit_a(q, xa);
      if (q + 1 < nkb) emit_a(q + 1, xb);
    }
  } else {
    // ---- MMA warpgroup g (lanes 64 g .. 64 g + 63); thread 0 of warpgroup 0 also bulk-copies the D^T tiles ----------
    // Segmented accumulation: the accumulator is drained into the CTA's workspace slot every SEG_KB k-blocks
    // (240 MMAs) and the segment sums are added up there with ordinary round-to-nearest fp32 adds, which bounds the
    // error growth of a single long accumulation chain.
    const int g = warp / 4 - 1;
    if (g >= nact) return;                    // lanes beyond the job's real ones: no MMAs, no drain
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(WG_REGS_MMA));
    const int t = tid - (g + 1) * 128, w = t >> 5, l = t & 31;
    const bool issuer = g == 0 && t == 0;
    // workspace block layout [column n][lane ka]
    float* out = wsj + g * WG_HALF + 16 * w + (l >> 2);
    long long* prof = (issuer && k.prof != nullptr && sp == 0 && i == 0) ? k.prof + (size_t)jslot * 1024 : nullptr;
    if (prof) { prof[0] = clock64(); prof[3] = kind | (d.N << 8); }
    auto fetch = [&](int q, int st) {
      const int kb = kb0 + q;
      const int tt = kb / bpt, rb = kb - tt * bpt;
      const uint8_t* tile = reinterpret_cast<const uint8_t*>(d.BT + nmarl_tc_tile_offset(d.tile_rows, tt, N_agents, bpt, i, rb));
      uint8_t* dst = bst + (size_t)st * 2 * tile_bytes;         // the raw tile lands in the hi half of the stage
      tc::mbar_arrive_expect_tx(&b_full[st], tile_bytes);
      tc::bulk_g2s(dst, tile + (size_t)d.n_row0 * 128, tile_bytes, &b_full[st]);
    };
    if (issuer)
      for (int q = 0; q < S && q < nkb; ++q) fetch(q, q);
    float acc[128];
#pragma unroll
    for (int j = 0; j < 128; ++j) acc[j] = 0.f;
    auto drain = [&](bool rmw) {
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        if (8 * j < d.N) {
          const int n = 8 * j + 2 * (l & 3);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            float* o = out + (size_t)(n + (e & 1)) * 128 + 8 * (e >> 1);
            *o = rmw ? *o + acc[4 * j + e] : acc[4 * j + e];
          }
        }
      }
    };
    RingPos as, bs;
    for (int q = 0; q < nkb; ++q) {
      const bool seg_first = (q % SEG_KB) == 0;
      uint8_t* b = bst + (size_t)bs.idx * 2 * tile_bytes;
      tc::mbar_wait(&b_split[bs.idx], bs.ph, k.err, 33);      // landed and split (A producers)
      if (prof && q < 300) prof[4 + 3 * q] = clock64();
      tc::mbar_wait(&a_full[as.idx], as.ph, k.err, 32);
      if (prof && q < 300) prof[5 + 3 * q] = clock64();
      uint8_t* a = ast + (size_t)as.idx * WG_A_SLOT + g * (WG_A_TILE / 2);
      tc::wgmma_fence();
      tc::wgmma_kblock_3x(d.N, acc, tc::smem_desc_sw128(a), tc::smem_desc_sw128(a + WG_A_TILE), tc::smem_desc_sw128(b),
                          tc::smem_desc_sw128(b + tile_bytes), 4, seg_first);
      tc::wgmma_commit();
      tc::wgmma_wait_all();
      if (prof && q < 300) prof[6 + 3 * q] = clock64();
      if (l == 0) { tc::mbar_arrive(&a_empty[as.idx]); tc::mbar_arrive(&b_empty[bs.idx]); }
      if (issuer && q + S < nkb) {
        tc::mbar_wait(&b_empty[bs.idx], bs.ph, k.err, 34);         // every active warpgroup has retired k-block q
        fetch(q + S, bs.idx);
      }
      as.next(AS); bs.next(S);
      if ((q + 1) % SEG_KB == 0 || q + 1 == nkb) drain(q >= SEG_KB);
    }
    if (nkb == 0) drain(false);                // acc is zero: the reduce reads every real lane of the block
    if (prof) { prof[1] = min(nkb, 300); prof[2] = clock64(); }
  }
}

// fixed-order reduce over the row splits + scatter into the flat gradient buffer
__global__ void __launch_bounds__(256) tc_wgrad_reduce_kernel(const __grid_constant__ nmarl_model m, const __grid_constant__ TcWgK k,
                                                             float* __restrict__ grads) {
  const int jslot = blockIdx.y, i = blockIdx.z, kind = k.jobs[jslot];
  const JobDesc d = job_desc(m, k, kind, i);
  const nmarl_agent& ag = m.agent[i];
  const int lanes = d.ka_cnt + (d.ones ? 1 : 0) + d.p_cnt;
  const int total = 128 * d.N;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    const int ln = e & 127, n = e >> 7;                      // partial blocks are [column n][lane]: coalesced over lanes
    if (ln >= lanes) continue;
    float s = 0.f;
    for (int sp = 0; sp < k.splits; ++sp) s += k.ws[k.ws_off[jslot] + (((size_t)sp * m.n_agent + i) * d.N + n) * 128 + ln];
    if (kind == J_GATE0 || kind == J_GATE1) grads[ag.o_wxh + (size_t)(128 * (kind - J_GATE0) + ln) * NG + n] = s;
    else if (kind == J_ENC_X) {
      if (ln < d.ka_cnt) { if (n < NH) grads[ag.o_w_ob + ln * NH + n] = s; }
      else if (ln > d.ka_cnt) { if (n >= NH && n < 2 * NH) grads[ag.o_w_fp + (ln - d.ka_cnt - 1) * NH + n - NH] = s; }   // fingerprint lanes
      else if (n < NH) grads[ag.o_b_ob + n] = s;                                       // ones lane: biases
      else if (m.variant == NMARL_NC && n < 2 * NH) grads[ag.o_b_fp + n - NH] = s;
      else if (ag.o_b_msg >= 0) grads[ag.o_b_msg + n - ((m.variant == NMARL_NC) ? 2 * NH : NH)] = s;
    } else grads[ag.o_w_msg + (size_t)(128 * (kind - J_ENC_M0) + ln) * NH + n] = s;
  }
}

// gate bias gradient: fixed-order reduce of the per-tile partial sums the backward cell kernel left in sv_dz
// ([t][agent][32-row tile][256]); one CTA per (32 columns, agent), 8 strided partial chains per column + an ordered tail
__global__ void __launch_bounds__(256) gate_bias_reduce_kernel(const __grid_constant__ nmarl_model m, const float* __restrict__ part,
                                                              int tiles, int T, float* __restrict__ grads) {
  __shared__ float red[8][32];
  const int c = threadIdx.x & 31, p = threadIdx.x >> 5, col = blockIdx.x * 32 + c, i = blockIdx.y;
  const int n = T * tiles;
  float s = 0.f;
  for (int e = p; e < n; e += 8) {
    const int t = e / tiles, tile = e - t * tiles;
    s += part[(((size_t)t * m.n_agent + i) * tiles + tile) * NG + col];
  }
  red[p][c] = s;
  __syncthreads();
  if (p == 0) {
    float tsum = 0.f;
    for (int w = 0; w < 8; ++w) tsum += red[w][c];
    grads[m.agent[i].o_b + col] = tsum;
  }
}

NMARL_PARAMS_FIT(nmarl_model, TcWgK);                                            // tc_wgrad_kernel
NMARL_PARAMS_FIT(nmarl_model, TcWgK, float*);                                    // tc_wgrad_reduce_kernel
NMARL_PARAMS_FIT(nmarl_model, const float*, int, int, float*);                   // gate_bias_reduce_kernel

int job_list(const nmarl_model* m, int* jobs) {
  int n = 0;
  jobs[n++] = J_GATE0;
  if (m->s_dim + NH > 128) jobs[n++] = J_GATE1;
  jobs[n++] = J_ENC_X;
  // (the fingerprint encoder shares the obs-encoder job: its few features sit on spare lanes of that tile)
  if (m->variant != NMARL_IA2C) {
    jobs[n++] = J_ENC_M0;
    if (m->km_pad > 128) jobs[n++] = J_ENC_M1;
  }
  return n;
}
int job_N(const nmarl_model* m, int kind) {
  if (kind == J_GATE0 || kind == J_GATE1) return 256;
  if (kind == J_ENC_X) return nmarl_tc_ndp(m);
  return 64;
}

}  // namespace

int nmarl_tc_ndp(const nmarl_model* m) { return m->variant == NMARL_NC ? 192 : (m->variant == NMARL_IA2C ? 64 : 128); }

int nmarl_tc_wgrad_splits(int n_agent) {
  int s = 33;                                   // 4 jobs x 33 x 8 agents = 1056 CTAs = 8 waves of 132 SMs
  while (4 * s * n_agent > 132 * 8 && s > 1) s = (s + 1) / 2;
  return s;
}

int64_t nmarl_tc_wgrad_ws_floats(const nmarl_model* m) {
  int jobs[J_COUNT];
  const int nj = job_list(m, jobs);
  int64_t tot = 0;
  for (int j = 0; j < nj; ++j) tot += (int64_t)nmarl_tc_wgrad_splits(m->n_agent) * m->n_agent * 128 * job_N(m, jobs[j]);
  return tot;
}

int nmarl_tc_launch_wgrads(const nmarl_model* m, int B, int T, const float* sv_sh, const float* sv_xin, const float* dzT,
                           const float* dpT, const float* sv_dz, float* ws, float* grads, int* err, cudaStream_t st,
                           cudaStream_t st_bias, void** ev_wgrad, const float* h_seq, const float* done_pre) {
  TcWgK k{};
  k.B = B; k.T = T; k.splits = nmarl_tc_wgrad_splits(m->n_agent); k.ndp = nmarl_tc_ndp(m);
  k.sv_sh = sv_sh; k.sv_xin = sv_xin; k.dzT = dzT; k.dpT = dpT; k.ws = ws; k.err = err;
  k.h_seq = h_seq; k.done_pre = done_pre; k.prof = g_nmarl_prof;
  k.n_jobs = job_list(m, k.jobs);
  long long off = 0;
  for (int j = 0; j < k.n_jobs; ++j) { k.ws_off[j] = off; off += (long long)k.splits * m->n_agent * 128 * job_N(m, k.jobs[j]); }
  static bool configured = false;
  if (!configured) {
    NMARL_CUDA(cudaFuncSetAttribute(tc_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WG_SMEM));
    configured = true;
  }
  // independent of the GEMM jobs; the backward cell kernel leaves one partial per 32 env rows
  gate_bias_reduce_kernel<<<dim3(NG / 32, m->n_agent), 256, 0, st_bias>>>(*m, sv_dz, B / 32, T, grads);
  NMARL_LAUNCH_CHECK();
  if (ev_wgrad) NMARL_CUDA(cudaEventRecord((cudaEvent_t)ev_wgrad[0], st));
  const dim3 grid(k.splits, k.n_jobs, m->n_agent);                   // one CTA per (row split, 128-lane job tile, agent)
  tc_wgrad_kernel<<<grid, WG_THREADS, WG_SMEM, st>>>(*m, k);
  NMARL_LAUNCH_CHECK();
  if (ev_wgrad) NMARL_CUDA(cudaEventRecord((cudaEvent_t)ev_wgrad[1], st));
  NMARL_DBG_SYNC(st, "tc_wgrad_kernel");
  tc_wgrad_reduce_kernel<<<dim3(64, k.n_jobs, m->n_agent), 256, 0, st>>>(*m, k, grads);
  NMARL_LAUNCH_CHECK();
  NMARL_DBG_SYNC(st, "tc_wgrad_reduce");
  return 0;
}
