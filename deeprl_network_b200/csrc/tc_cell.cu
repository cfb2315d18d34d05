// tc_cell.cu -- tensor-core (wgmma) version of the fused forward cell (K2..K6):
// every GEMM of the step (obs / fingerprint / message encoders and the LSTM gate GEMM) runs as
// 3xTF32 wgmma with FP32 accumulators; CUDA cores only do the gathers and the elementwise epilogues.
//
// One CTA = 64 envs of one agent (wgmma M = 64).  384 threads:
//   warps 0-7  "row threads": 4 warp-sets x 2 warps; a thread of set s in warp half h owns env row
//              r = 32 h + lane and the column slice s of it.  They gather the row's inputs, split them hi/lo
//              and store them as the A operand (a 128B-swizzled shared-memory ring), read the finished GEMM
//              results back from the accumulator staging area, apply bias/activation, feed them to the gate
//              GEMM, and finally run the LSTM cell update, the heads, softmax and sampling for their row.
//   warps 8-11 MMA warpgroup: 3 wgmma per 8-deep k-step (hi*hi + hi*lo + lo*hi) into a register accumulator;
//              each finished GEMM is stored to the staging area (tc_row.cuh).  Its thread 0 also streams the
//              pre-packed, 128B-swizzled [hi | lo] weight tiles, one cp.async.bulk (TMA engine) per 32-wide
//              k-block, into a 2-stage shared-memory ring (mbarrier tx).
// Staging area (64 rows x 256 columns): the encoder GEMMs land in 64-column blocks of it and are consumed before
// the gate GEMM overwrites it.
//
// Same math, same argument block and same outputs as cell_fwd.cu (FP32 FFMA); used when
// B % 128 == 0 and packed weights are supplied.  Restates the same reference lines as cell_fwd.cu.
#include "cell_common.cuh"
#include "tc_row.cuh"

int nmarl_launch_pack_b(const float* W, int ldw, int K, int n0, int nrows, float* out, cudaStream_t st);

namespace {

using namespace tcrow;

template <int VAR, int MODE, int HW>
__global__ void __launch_bounds__(TC_THREADS, 1) tc_cell_fwd_kernel(const __grid_constant__ nmarl_model m,
                                                                    const __grid_constant__ FwdK k) {
  constexpr bool FM = VAR != NMARL_DIAL;                           // state layout: DIAL's message kernels are env-major
  constexpr bool SAVE = (MODE == MODE_PS);                         // store activations for BPTT
  constexpr bool SAMPLE = (MODE == MODE_P || MODE == MODE_PS);     // p-call: sample actions
  static_assert(HW <= EW, "a set's HW partial head sums live in its EW gate-f staging columns");
  extern __shared__ uint8_t smem_raw[];
  const Smem sm = smem_map(smem_raw);

  const nmarl_fwd_args& a = k.a;
  const int i = blockIdx.y;
  const nmarl_agent& ag = m.agent[i];
  const int B = a.B, b0 = blockIdx.x * ROWS;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_a = m.n_a, SD = m.s_dim;
  const float* __restrict__ P = a.params;
  const int Kx = ag.x_nsrc * ag.x_w;

  if (tid == 0) {
    init_barriers(sm);
    // ---- k-block schedule shared by the three roles: all encoder GEMMs first (each into its own 64-column
    // block of the accumulator region, one completion barrier), then the gate GEMM over [s | h^] ----------------
    // An agent without neighbours has zero-width fingerprint / message operands: they get no k-block (and no packed
    // tiles to copy), and the row threads feed relu(0 + b) for them, as the FFMA kernel does.
    SchedBuilder sb(sm);
    sb.gemm(ag.tp_x, 64, Kx, ACC_COL, DONE_NONE);                                           // X (Kx <= 32 on this path)
    if (VAR == NMARL_NC) sb.gemm(ag.tp_p, 64, ag.n_nbr * n_a, ACC_COL + 64, DONE_NONE);     // no neighbours: K = 0
    if (VAR != NMARL_IA2C) {
      const int KM = (VAR == NMARL_IC3) ? NH : NH * ag.n_nbr;
      sb.gemm(ag.tp_m, 64, KM, (VAR == NMARL_NC) ? ACC_COL + 128 : ACC_COL + 64, DONE_NONE);
    }
    sm.seg[sb.ns - 1].done = DONE_ENC;                  // the last encoder GEMM actually scheduled completes enc_full
    sb.gemm(ag.tp_g, 256, SD + NH, ACC_COL, DONE_ACC);
    if (VAR == NMARL_DIAL && MODE != MODE_V) sb.gemm(ag.tp_mfc, 64, NH, ACC_COL, DONE_ENC);
    sb.finish();
  }
  __syncthreads();
  // PDL: the prologue above overlapped the tail of the previous kernel of the stream; from here on the kernel reads
  // what that kernel (env step / previous cell call) wrote.
  tc::pdl_launch_dependents();
  tc::pdl_wait();

  if (warp < MMA_WARP0) {
    // =================================== row threads ===================================================
    RowCtx c;
    const int set = warp / ROW_WARPS, rh = warp % ROW_WARPS, r = rh * 32 + lane;
    c.a_ring = sm.ast; c.acc = sm.acc; c.r = (uint32_t)r;
    c.a_full = sm.a_full; c.a_empty = sm.a_empty; c.enc_full = sm.enc_full; c.q = 0; c.e = 0; c.set = set; c.err = a.tc_err;
    const int b = b0 + r;
    const size_t row = (size_t)i * B + b;
    const float nd = 1.0f - a.done[b];
    const int LDI = m.kx_pad + m.kp_pad + m.km_pad;
    // saved activations are feature-major on this path: [agent][feature][env]
    float* xin_fm = SAVE ? a.sv_xin + (size_t)i * LDI * B : nullptr;
    float* sh_fm = SAVE ? a.sv_sh + (size_t)i * (SD + NH) * B : nullptr;
    float* enc_fm = (SAVE && a.sv_enc) ? a.sv_enc + (size_t)i * 128 * B : nullptr;
    float* gates_fm = SAVE ? a.sv_gates + (size_t)i * NG * B : nullptr;
    long long* prof = (k.prof != nullptr && blockIdx.x == 0 && blockIdx.y == 1 && tid == 0) ? k.prof : nullptr;
    int pi_ = 0;
#define STAMP() do { if (prof) prof[pi_++] = clock64(); } while (0)
    STAMP();
    const int c0 = set * W;             // this thread's columns inside every 32-wide input k-block
    const int e0 = set * EW;            // this thread's hidden units / encoder columns

    // ---- gather every encoder input of this thread up front (all loads in flight together) ------------------
    const int inv_xw = 65536 / ag.x_w + 1, inv_na = 65536 / n_a + 1;    // exact floor(kk / d) for kk < 32, d <= 32
    float xv[W];
#pragma unroll
    for (int j = 0; j < W; ++j) {
      const int kk = c0 + j;
      float val = 0.f;
      if (kk < Kx) {
        const int s = (kk * inv_xw) >> 16, f = kk - s * ag.x_w;     // kk / x_w for kk < 32 without an integer division
        val = a.obs[((size_t)ag.x_src[s] * B + b) * m.obs_stride + f];
      }
      xv[j] = val;
    }
    float pv[W];
    if (VAR == NMARL_NC) {
      const int Kp = ag.n_nbr * n_a;
#pragma unroll
      for (int j = 0; j < W; ++j) {
        const int kk = c0 + j;
        float val = 0.f;
        if (kk < Kp) {
          const int s = (kk * inv_na) >> 16, f = kk - s * n_a;
          val = a.fp[((size_t)ag.nbr[s] * B + b) * n_a + f];
        }
        pv[j] = val;
      }
    }
    constexpr int NPRE = 2;                      // neighbours whose messages are prefetched into registers
    float mv[NPRE][2][W];
    if (VAR == NMARL_NC || VAR == NMARL_DIAL) {
      const float* src = (VAR == NMARL_NC) ? a.h_in : a.msg_in;          // messages: UN-masked (utils.py:182-183)
#pragma unroll
      for (int s = 0; s < NPRE; ++s) {
        if (s < ag.n_nbr) {
#pragma unroll
          for (int hb = 0; hb < 2; ++hb) ld_state<FM, W>(src, (size_t)ag.nbr[s], b, hb * 32 + c0, B, mv[s][hb]);
        }
      }
    }
    if (VAR == NMARL_IC3) {                                               // mean of the neighbours' h (utils.py:395)
      const float nn = (float)ag.n_nbr;
#pragma unroll
      for (int hb = 0; hb < 2; ++hb) {
#pragma unroll
        for (int j = 0; j < W; ++j) mv[0][hb][j] = 0.f;
        for (int s = 0; s < ag.n_nbr; ++s) {
          float w8[W];
          ld_state<FM, W>(a.h_in, (size_t)ag.nbr[s], b, hb * 32 + c0, B, w8);
#pragma unroll
          for (int j = 0; j < W; ++j) mv[0][hb][j] += w8[j];
        }
#pragma unroll
        for (int j = 0; j < W; ++j) mv[0][hb][j] /= nn;
      }
    }
    float hv[2][W];                                                       // own h, done-masked (utils.py:189-190)
#pragma unroll
    for (int hb = 0; hb < 2; ++hb) {
      ld_state<FM, W>(a.h_in, (size_t)i, b, hb * 32 + c0, B, hv[hb]);
#pragma unroll
      for (int j = 0; j < W; ++j) hv[hb][j] *= nd;
    }
    STAMP();
    // ---- encoder GEMMs: A chunks back to back, one completion wait ----------------------------------------------
    const int xm0 = m.kx_pad + m.kp_pad;
    // kx_pad / kp_pad are multiples of 4, the column slices 8 wide: e.g. the 25 IA2C inputs on the 5x5 grid pad to 28,
    // and features 28..31 of the last slice would land on the next section (or the next agent's row of sv_xin)
    if (SAVE && c0 < m.kx_pad) st_fm<W>(xin_fm, c0, B, b, xv, m.kx_pad - c0);
    produce_in(c, xv);
    if (VAR == NMARL_NC) {
      if (SAVE && c0 < m.kp_pad) st_fm<W>(xin_fm, m.kx_pad + c0, B, b, pv, m.kp_pad - c0);
      if (ag.n_nbr > 0) produce_in(c, pv);              // no fingerprint k-block without neighbours (schedule above)
    }
    if (VAR == NMARL_IC3) {
#pragma unroll
      for (int hb = 0; hb < 2; ++hb) {
        if (SAVE) st_fm<W>(xin_fm, xm0 + hb * 32 + c0, B, b, mv[0][hb]);
        produce_in(c, mv[0][hb]);
      }
    } else if (VAR != NMARL_IA2C) {
      const float* src = (VAR == NMARL_NC) ? a.h_in : a.msg_in;
      for (int s = 0; s < ag.n_nbr; ++s) {
#pragma unroll
        for (int hb = 0; hb < 2; ++hb) {
          float t[W];
          if (s < NPRE) {
#pragma unroll
            for (int j = 0; j < W; ++j) t[j] = (s == 0) ? mv[0][hb][j] : mv[NPRE - 1][hb][j];
          } else {
            ld_state<FM, W>(src, (size_t)ag.nbr[s], b, hb * 32 + c0, B, t);
          }
          // NeurComm: m~ is a plain copy of the neighbours' h_seq[t]; the weight-gradient kernel reads it from there
          // (tc_wgrad.cu), so it is not saved a second time
          if (SAVE && VAR != NMARL_NC) st_fm<W>(xin_fm, xm0 + s * NH + hb * 32 + c0, B, b, t);
          produce_in(c, t);
        }
      }
      if (SAVE && VAR != NMARL_NC) {
        float z[W];
#pragma unroll
        for (int j = 0; j < W; ++j) z[j] = 0.f;
        for (int q = ag.n_nbr * 2; q < m.km_pad / 32; ++q) st_fm<W>(xin_fm, xm0 + q * 32 + c0, B, b, z);
      }
    }
    STAMP();
    enc_wait(c);
    STAMP();
    // ---- encoder epilogues -> s, fed to the gate GEMM ---------------------------------------------------------------
    float s0[EW];
    enc_load(c, ACC_COL, s0);
    bias_act(s0, P + ag.o_b_ob + e0, VAR == NMARL_IC3 ? 1 : 0);
    if (SAVE && (VAR == NMARL_IC3 || VAR == NMARL_DIAL)) st_fm<EW>(enc_fm, e0, B, b, s0);
    // an encoder GEMM that was not scheduled (no neighbours) contributes 0 before its bias
    auto enc_load_or_0 = [&](bool present, uint32_t col, float (&v)[EW]) {
      if (present) { enc_load(c, col, v); return; }
#pragma unroll
      for (int j = 0; j < EW; ++j) v[j] = 0.f;
    };
    if (VAR == NMARL_NC) {
      float s1[EW], s2[EW];
      enc_load_or_0(ag.n_nbr > 0, ACC_COL + 64, s1);
      enc_load_or_0(ag.n_nbr > 0, ACC_COL + 128, s2);
      bias_act(s1, P + ag.o_b_fp + e0, 0);
      bias_act(s2, P + ag.o_b_msg + e0, 0);
      if (SAVE) { st_fm<EW>(sh_fm, e0, B, b, s0); st_fm<EW>(sh_fm, NH + e0, B, b, s1); st_fm<EW>(sh_fm, 2 * NH + e0, B, b, s2); }
      produce_act(c, s0);
      produce_act(c, s1);
      produce_act(c, s2);
    } else if (VAR == NMARL_IA2C) {
      if (SAVE) st_fm<EW>(sh_fm, e0, B, b, s0);
      produce_act(c, s0);
    } else {
      float s1[EW];
      enc_load_or_0(VAR == NMARL_IC3 || ag.n_nbr > 0, ACC_COL + 64, s1);
      if (VAR == NMARL_IC3) {                                            // s = tanh(..) + m W_msg + b  (utils.py:400)
        bias_act(s1, P + ag.o_b_msg + e0, 2);
#pragma unroll
        for (int j = 0; j < EW; ++j) s0[j] += s1[j];
      } else {                                                           // DIAL: relu + relu + onehot(argmax p_i)
        // without a message encoder (o_b_msg < 0, see nmarl.h) s is the observation encoder alone: s1 stays 0, no one-hot
        const bool has_msg = ag.o_b_msg >= 0;
        if (has_msg) bias_act(s1, P + ag.o_b_msg + e0, 0);
        if (SAVE) st_fm<EW>(enc_fm, NH + e0, B, b, s1);
        int am = has_msg ? 0 : -1;
        if (has_msg) {
          const float* pr = a.fp + row * n_a;
          float best = pr[0];
          for (int cc = 1; cc < n_a; ++cc) { const float pvv = pr[cc]; if (pvv > best) { best = pvv; am = cc; } }
        }
#pragma unroll
        for (int j = 0; j < EW; ++j) s0[j] = (s0[j] + s1[j]) + ((e0 + j) == am ? 1.0f : 0.0f);
      }
      if (SAVE) st_fm<EW>(sh_fm, e0, B, b, s0);
      produce_act(c, s0);
    }
#pragma unroll
    for (int hb = 0; hb < 2; ++hb) {
      // outside DIAL h^ = (1 - done) * h_seq[t] is re-derived by tc_wgrad from the feature-major state sequence
      if (SAVE && VAR == NMARL_DIAL) st_fm<W>(sh_fm, SD + hb * 32 + c0, B, b, hv[hb]);
      produce_in(c, hv[hb]);
    }
    STAMP();
    // ---- LSTM cell update for hidden units [e0, e0 + EW), 8 at a time; partial head sums -----------------------
    tc::mbar_wait(sm.acc_full, 0, a.tc_err, 13);
    STAMP();
    float logit[HW];
#pragma unroll
    for (int cc = 0; cc < HW; ++cc) logit[cc] = 0.f;
    float v = 0.f;
#pragma unroll 1
    for (int u0 = e0; u0 < e0 + EW; u0 += 8) {
      float gi[8], gf[8], go[8], gu[8];
      acc_ld8(c, ACC_COL + 0 * NH + u0, gi);
      acc_ld8(c, ACC_COL + 1 * NH + u0, gf);
      acc_ld8(c, ACC_COL + 2 * NH + u0, go);
      acc_ld8(c, ACC_COL + 3 * NH + u0, gu);
      STAMP();
      float cn[8], hn[8], cpv[8];
      ld_state<FM, 8>(a.c_in, (size_t)i, b, u0, B, cpv);
      // MUFU budget: the SFU (16 lanes/clk/SM) bounds this loop, so reciprocals are shared pairwise:
      // 1/(1+a), 1/(1+b) from ONE rcp of (1+a)(1+b)  ->  5 ex2 + 2.5 rcp per hidden unit instead of 5 + 5
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const float4 bi = __ldg(reinterpret_cast<const float4*>(P + ag.o_b + 0 * NH + u0) + q);
        const float4 bf = __ldg(reinterpret_cast<const float4*>(P + ag.o_b + 1 * NH + u0) + q);
        const float4 bo = __ldg(reinterpret_cast<const float4*>(P + ag.o_b + 2 * NH + u0) + q);
        const float4 bu = __ldg(reinterpret_cast<const float4*>(P + ag.o_b + 3 * NH + u0) + q);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int x = 4 * q + j;
          const float di = 1.0f + __expf(fminf(-(gi[x] + f4get(bi, j)), 40.0f));
          const float df = 1.0f + __expf(fminf(-(gf[x] + f4get(bf, j)), 40.0f));
          const float dO = 1.0f + __expf(fminf(-(go[x] + f4get(bo, j)), 40.0f));
          const float du = 1.0f + __expf(fminf(-2.0f * (gu[x] + f4get(bu, j)), 40.0f));
          const float r1 = frcp_(di * df), r2 = frcp_(dO * du);
          gi[x] = r1 * df;                          // sigmoid(i)
          gf[x] = r1 * di;                          // sigmoid(f)
          go[x] = r2 * du;                          // sigmoid(o)
          gu[x] = fmaf(2.0f, r2 * dO, -1.0f);       // tanh(u)
          cn[x] = gf[x] * (cpv[x] * nd) + gi[x] * gu[x];
        }
      }
#pragma unroll
      for (int x = 0; x < 8; x += 2) {              // tanh(c) for two units from one reciprocal
        const float d0 = 1.0f + __expf(fminf(-2.0f * cn[x], 40.0f)), d1 = 1.0f + __expf(fminf(-2.0f * cn[x + 1], 40.0f));
        const float r = frcp_(d0 * d1);
        hn[x] = go[x] * fmaf(2.0f, r * d1, -1.0f);
        hn[x + 1] = go[x + 1] * fmaf(2.0f, r * d0, -1.0f);
      }
      STAMP();
      if (MODE != MODE_V) {
        st_state<FM, 8>(a.c_out, (size_t)i, b, u0, B, cn);
        st_state<FM, 8>(a.h_out, (size_t)i, b, u0, B, hn);
      }
      if (SAVE) {
        st_fm<8>(gates_fm, 0 * NH + u0, B, b, gi); st_fm<8>(gates_fm, 1 * NH + u0, B, b, gf);
        st_fm<8>(gates_fm, 2 * NH + u0, B, b, go); st_fm<8>(gates_fm, 3 * NH + u0, B, b, gu);
      }
      STAMP();
      if (MODE != MODE_V) {
        if (n_a == 4) {
#pragma unroll
          for (int x = 0; x < 8; ++x) {
            const float4 w4 = __ldg(reinterpret_cast<const float4*>(P + ag.o_pi_w) + u0 + x);
            logit[0] = fmaf(hn[x], w4.x, logit[0]); logit[1] = fmaf(hn[x], w4.y, logit[1]);
            logit[2] = fmaf(hn[x], w4.z, logit[2]); logit[3] = fmaf(hn[x], w4.w, logit[3]);
          }
        } else {
          // one logit at a time (each still sums its 8 units in order): with the units outer, ptxas hoisted all
          // HW x 8 weight loads and the HW = 16 saving instantiations spilled
#pragma unroll
          for (int cc = 0; cc < HW; ++cc)
#pragma unroll
            for (int x = 0; x < 8; ++x)
              if (cc < n_a) logit[cc] = fmaf(hn[x], __ldg(P + ag.o_pi_w + (u0 + x) * n_a + cc), logit[cc]);
        }
      }
      if (!SAMPLE) {
        const float4 v0 = __ldg(reinterpret_cast<const float4*>(P + ag.o_v_w + u0)), v1 = __ldg(reinterpret_cast<const float4*>(P + ag.o_v_w + u0) + 1);
        v = fmaf(hn[0], v0.x, v); v = fmaf(hn[1], v0.y, v); v = fmaf(hn[2], v0.z, v); v = fmaf(hn[3], v0.w, v);
        v = fmaf(hn[4], v1.x, v); v = fmaf(hn[5], v1.y, v); v = fmaf(hn[6], v1.z, v); v = fmaf(hn[7], v1.w, v);
      }
      STAMP();
      if (VAR == NMARL_DIAL && MODE != MODE_V) {          // stash h' for the sender-side message fc below
#pragma unroll
        for (int x = 0; x < 8; ++x) s0[(u0 - e0) + x] = hn[x];
      }
    }
    if (VAR == NMARL_DIAL && MODE != MODE_V) produce_act(c, s0);

    // ---- heads: combine the NSET partial sums of a row in fixed order, then softmax / sampling ---------------
    // The partial sums of set s go to staging columns [NH + s*EW, +HW) of the row (HW - 1 logits, then v): gate-f
    // cells that only this thread has read, and that the DIAL message GEMM (columns [0, NH)) does not overwrite.
    {
      float* hp = sm.acc;
#pragma unroll
      for (int cc = 0; cc < HW - 1; ++cc) hp[acc_idx(r, NH + e0 + cc)] = logit[cc];
      hp[acc_idx(r, NH + e0 + HW - 1)] = v;
    }
    STAMP();
    row_barrier();
    STAMP();
    if (set == 0) {
#pragma unroll
      for (int cc = 0; cc < HW; ++cc) logit[cc] = 0.f;
      v = 0.f;
#pragma unroll
      for (int s = 0; s < NSET; ++s) {
        const float* hp = sm.acc;
#pragma unroll
        for (int cc = 0; cc < HW - 1; ++cc) logit[cc] += hp[acc_idx(r, NH + s * EW + cc)];
        v += hp[acc_idx(r, NH + s * EW + HW - 1)];
      }
      float pi[HW];
      if (MODE != MODE_V) {
        float mx = -3.0e38f;
#pragma unroll
        for (int cc = 0; cc < HW; ++cc)
          if (cc < n_a) { logit[cc] += __ldg(P + ag.o_pi_b + cc); mx = fmaxf(mx, logit[cc]); }
        float se = 0.f;
#pragma unroll
        for (int cc = 0; cc < HW; ++cc)
          if (cc < n_a) { pi[cc] = expf(logit[cc] - mx); se += pi[cc]; } else pi[cc] = 0.f;
#pragma unroll
        for (int cc = 0; cc < HW; ++cc)
          if (cc < n_a) { pi[cc] = pi[cc] / se; if (a.pi != nullptr) a.pi[row * n_a + cc] = pi[cc]; }
      }
      if (SAMPLE && a.action != nullptr && a.sample_mode != NMARL_SAMPLE_NONE) {
        int act = 0;
        if (a.sample_mode == NMARL_SAMPLE_GREEDY) {
          float best = pi[0];
#pragma unroll
          for (int cc = 1; cc < HW; ++cc) if (cc < n_a && pi[cc] > best) { best = pi[cc]; act = cc; }
        } else {
          double u;
          if (a.sample_mode == NMARL_SAMPLE_UNIFORM) u = a.uniforms[row];
          else u = philox_u01(a.rng[0], a.rng[1] + a.rng_offset, nmarl_sample_lane(a, i, b), 0x41435431u);
          double cdf[HW];
          double s = 0.0;
#pragma unroll
          for (int cc = 0; cc < HW; ++cc) { if (cc < n_a) s += (double)pi[cc]; cdf[cc] = s; }
          if (a.sample_mode == NMARL_SAMPLE_UNIFORM) {
            // host-supplied uniforms: np.random.choice's rule verbatim (cdf /= cdf[-1]; searchsorted(cdf, u, 'right'))
#pragma unroll
            for (int cc = 0; cc < HW; ++cc) if (cc < n_a) act += ((cdf[cc] / s) <= u) ? 1 : 0;
          } else {
            // device Philox stream (no NumPy stream to reproduce): the same inverse-cdf draw without the four fp64
            // divisions -- they are the longest dependent chain of the kernel's tail
            const double us = u * s;
#pragma unroll
            for (int cc = 0; cc < HW; ++cc) if (cc < n_a) act += (cdf[cc] <= us) ? 1 : 0;
          }
          act = min(act, n_a - 1);
        }
        a.action[row] = act;
      }
      if (!SAMPLE) {
        for (int s = 0; s < ag.n_nbr; ++s) v += __ldg(P + ag.o_v_w + NH + s * n_a + a.act_in[(size_t)ag.nbr[s] * B + b]);
        v += __ldg(P + ag.o_v_b);
        if (a.v != nullptr) a.v[row] = v;
      }
    }
    if (VAR == NMARL_DIAL && MODE != MODE_V) {            // msg' = relu(h' W_mfc + b)   (utils.py:563-566)
      float mo[EW];
      enc_wait(c);
      enc_load(c, ACC_COL, mo);
      bias_act(mo, P + ag.o_mfc_b + e0, 0);
      st_state<FM, EW>(a.msg_out, (size_t)i, b, e0, B, mo);
    }
    STAMP();
    if (prof) prof[31] = pi_;
  } else {
    // =================================== MMA warpgroup ===================================================
    mma_loop<MMA_PIPE | MMA_PARTIAL, 64, 256>(sm, a.wpack, a.tc_err);
  }
  __syncthreads();
}


NMARL_PARAMS_FIT(nmarl_model, FwdK);                                             // tc_cell_fwd_kernel

template <int VAR, int MODE, int HW>
int launch_tc_hw(const nmarl_model* m, const FwdK& k, cudaStream_t st) {
  auto kern = tc_cell_fwd_kernel<VAR, MODE, HW>;
  static bool configured = false;
  if (!configured) {
    NMARL_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_SMEM));
    configured = true;
  }
  dim3 grid(k.a.B / ROWS, m->n_agent);
  FwdK k2 = k;
  k2.prof = g_nmarl_prof;
  NMARL_CUDA(nmarl_launch(kern, grid, dim3(TC_THREADS), TC_SMEM, st, true, *m, k2));
  NMARL_LAUNCH_CHECK();
  return 0;
}

template <int VAR, int MODE>
int launch_tc(const nmarl_model* m, const FwdK& k, cudaStream_t st) {
  return nmarl_head_width(m->n_a) == 8 ? launch_tc_hw<VAR, MODE, 8>(m, k, st) : launch_tc_hw<VAR, MODE, 16>(m, k, st);
}

template <int VAR>
int launch_tc_mode(const nmarl_model* m, const FwdK& k, int mode, cudaStream_t st) {
  switch (mode) {
    case MODE_P: return launch_tc<VAR, MODE_P>(m, k, st);
    case MODE_V: return launch_tc<VAR, MODE_V>(m, k, st);
    default: return launch_tc<VAR, MODE_PS>(m, k, st);
  }
}

}  // namespace

bool nmarl_tc_fwd_supported(const nmarl_model* m, const nmarl_fwd_args* a) {
  if (a->wpack == nullptr || a->B % 128 != 0 || m->kx_pad > 32 || m->kp_pad > 32 || nmarl_n_h(*m) != NMARL_NH) return false;
  for (int i = 0; i < m->n_agent; ++i)
    if (m->agent[i].tp_g < 0 || m->agent[i].tp_x < 0) return false;
  return true;
}

int nmarl_tc_launch_fwd(const nmarl_model* m, const FwdK& k, int mode, cudaStream_t st) {
  switch (m->variant) {
    case NMARL_IA2C: return launch_tc_mode<NMARL_IA2C>(m, k, mode, st);
    case NMARL_NC: return launch_tc_mode<NMARL_NC>(m, k, mode, st);
    case NMARL_IC3: return launch_tc_mode<NMARL_IC3>(m, k, mode, st);
    case NMARL_DIAL: return launch_tc_mode<NMARL_DIAL>(m, k, mode, st);
  }
  nmarl_set_error("unknown variant %d", m->variant);
  return 1;
}

namespace {
// One launch packs every tensor-core operand of every agent: per 32-deep k-block a [hi | lo] pair of 128B-swizzled
// K-major tiles (see tc.cuh).  Job j of agent i (blockIdx.y = i * PACK_JOBS + j) is one matrix; the backward
// operands (transposed weights) are gathered straight from the parameters with transposed indexing, so no
// transposed copy is needed on this path.
enum { PJ_X = 0, PJ_P, PJ_M, PJ_G, PJ_GT, PJ_MT, PJ_MFC, PJ_MFCT, PACK_JOBS };
struct PackJob { int src, ld, K, N, transposed, dst; };     // operand element (k, n) = transposed ? W[n * ld + k] : W[k * ld + n]

__device__ __forceinline__ PackJob pack_job(const nmarl_model& m, int i, int j) {
  const nmarl_agent& ag = m.agent[i];
  const int SD = m.s_dim, Kx = ag.x_nsrc * ag.x_w;
  const int Km = (m.variant == NMARL_IC3) ? NH : ag.n_nbr * NH;
  PackJob p{0, 0, 0, 0, 0, -1};
  switch (j) {
    case PJ_X: p = PackJob{ag.o_w_ob, NH, Kx, NH, 0, ag.tp_x}; break;
    case PJ_P: if (m.variant == NMARL_NC) p = PackJob{ag.o_w_fp, NH, ag.n_nbr * m.n_a, NH, 0, ag.tp_p}; break;
    case PJ_M: if (m.variant != NMARL_IA2C && Km > 0) p = PackJob{ag.o_w_msg, NH, Km, NH, 0, ag.tp_m}; break;
    case PJ_G: p = PackJob{ag.o_wxh, NG, SD + NH, NG, 0, ag.tp_g}; break;
    case PJ_GT: p = PackJob{ag.o_wxh, NG, NG, SD + NH, 1, ag.tp_gT}; break;
    case PJ_MT: if (m.variant != NMARL_IA2C && Km > 0) p = PackJob{ag.o_w_msg, NH, NH, Km, 1, ag.tp_mT}; break;
    case PJ_MFC: if (m.variant == NMARL_DIAL) p = PackJob{ag.o_mfc_w, NH, NH, NH, 0, ag.tp_mfc}; break;
    case PJ_MFCT: if (m.variant == NMARL_DIAL) p = PackJob{ag.o_mfc_w, NH, NH, NH, 1, ag.tp_mfcT}; break;
  }
  return p;
}

__global__ void __launch_bounds__(256) pack_all_kernel(const __grid_constant__ nmarl_model m, const float* __restrict__ params,
                                                       float* __restrict__ wpack) {
  const int i = blockIdx.y / PACK_JOBS, j = blockIdx.y % PACK_JOBS;
  const PackJob p = pack_job(m, i, j);
  if (p.dst < 0 || p.K <= 0 || p.N <= 0) return;
  const float* W = params + p.src;
  const int nkb = (p.K + 31) / 32;
  const int total = nkb * p.N * 32;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    int n, kk, kb;
    if (p.transposed) { kk = idx & 31; n = (idx >> 5) % p.N; kb = idx / (32 * p.N); }      // consecutive threads -> consecutive k
    else { n = idx % p.N; kk = (idx / p.N) & 31; kb = idx / (p.N * 32); }                  // consecutive threads -> consecutive n
    const int k = kb * 32 + kk;
    float x = 0.f;
    if (k < p.K) x = p.transposed ? W[(size_t)n * p.ld + k] : W[(size_t)k * p.ld + n];
    float hi, lo;
    tc::split_tf32(x, hi, lo);
    char* tile = reinterpret_cast<char*>(wpack + p.dst) + (size_t)kb * 2 * p.N * 128;
    const uint32_t off = tc::sw128_offset((uint32_t)n, (uint32_t)kk);
    *reinterpret_cast<float*>(tile + off) = hi;
    *reinterpret_cast<float*>(tile + (size_t)p.N * 128 + off) = lo;
  }
}
NMARL_PARAMS_FIT(nmarl_model, const float*, float*);                             // pack_all_kernel
}  // namespace

extern "C" int nmarl_pack_weights(const nmarl_model* m, const float* params, float* wt, float* wpack, void* stream) {
  NMARL_CHECK(m && params && wt && wpack, "pack_weights: missing buffers");
  NMARL_CHECK(nmarl_n_h(*m) == NMARL_NH, "pack_weights: the tensor-core kernels need n_h = %d (got %d)", NMARL_NH, nmarl_n_h(*m));
  cudaStream_t st = (cudaStream_t)stream;
  pack_all_kernel<<<dim3(16, m->n_agent * PACK_JOBS), 256, 0, st>>>(*m, params, wpack);
  NMARL_LAUNCH_CHECK();
  // DIAL's message-gradient kernel reads the plain transposed copies (one launch for every agent)
  if (m->variant == NMARL_DIAL && nmarl_launch_transposes(m, NMARL_TJ_MSG | NMARL_TJ_MFC, params, wt, st)) return 1;
  return 0;
}
