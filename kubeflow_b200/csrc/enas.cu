// ENAS controller (Katib algorithm `enas`): the macro-search LSTM controller of ENAS, its REINFORCE training and its
// architecture draws.  FP64 restatement: oracle/enas_oracle.py.
//
// Design (DESIGN.md §"enas"):
// * The controller is one sequential chain: 2·L dependent LSTM cells per sampled arc, then the same chain backwards.  The
//   train kernel is ONE CTA of 512 threads that runs all T steps (sample, forward, backward through both cells of every
//   layer, weight gradients, Adam) with no host round trip.  A single CTA keeps every barrier an intra-SM bar.sync and lets
//   the parameters it updates be re-read through the same SM's L1, so no grid-wide synchronisation or cache coherence is
//   needed.
// * Parameters stay in global memory and stream through L1 / L2.  w_lstm at H = 128 is 2H × 4H FP32 = 512 KiB: more than
//   the register file (256 KiB) and the shared memory (227 KiB) of one SM, so neither holds it; at H <= 64 it is 128 KiB
//   and stays L1-resident across a step.  Recurrent state, gates and logits live in shared memory; the per-cell tensors
//   the backward pass needs go to a global scratch that stays in L2.
// * The sample kernel draws EN_SB arcs per CTA: the cell, logit, attention and anchor matvecs of those arcs read each
//   weight once and feed EN_SB FMAs (a small GEMM).
// * FP32 throughout (upstream's graph is float32).  Every sum has a fixed order (sequential loops, xor-butterfly warp
//   sums, fixed cross-warp trees), and there are no atomics: the same calls give bit-identical results.
// * Draws: Philox4x32-10 keyed by the seed, counter (draw counter lo, hi, arc, decision); u = (word 0 >> 8)·2^-24.  A
//   decision takes the first bin whose inclusive prefix sum of exp(s - max) exceeds u·total.
#include <algorithm>
#include <cmath>
#include <new>

#include "kbo_internal.cuh"
#include "kbo_rng.cuh"

#define EN_MAXL 64
#define EN_MAXH 128
#define EN_MAXOPS 4096
#define EN_MAXK 1024
#define EN_MAXT 10000
#define EN_NT 512            // threads per CTA, both kernels
#define EN_NW (EN_NT / 32)
#define EN_SB 4              // arcs per CTA in the sample kernel
#define EN_NSTAT 6           // per-step statistics: nll, ent, mean kl, loss, baseline, skip rate

struct EnCfg {
  int L, H, n_ops, A;                   // A = L(L+1)/2 decisions per arc
  int use_temp, use_tanh;
  float temp, tanh_c, ent_w, decay, lr, skip_target, skip_w;
  uint32_t k0, k1;                      // Philox key (seed)
  long long o_lstm, o_gemb, o_wemb, o_soft, o_w1, o_w2, o_v, n_par;
};

struct EnDev {                          // device-resident scalars of the controller
  float baseline;
  int err;
  long long step, draws;
};

struct EnBufs {                         // the train kernel's per-step tensors (one arc), global scratch
  float *XH;                            // (2L + 1) × 2H: [x, h_prev] of every cell; row 2L holds [0, h_final]
  float *CS;                            // (2L + 1) × H: c before every cell, then the final c
  float *GT;                            // 2L × 4H: post-activation gates i, f, o, g
  float *DZS;                           // 2L × 4H: gate pre-activation gradients
  float *Z;                             // L × n_ops: raw op logits, overwritten by their gradients
  float *PR;                            // L × n_ops: op probabilities
  float *ANC;                           // L × H: anchors (h after cell B of each layer)
  float *AW1;                           // L × H: anchor_l · w_attn_1
  float *TA;                            // L(L-1)/2 × H: tanh(anchor_w1_j + h·w_attn_2)
  float *Q;                             // L(L-1)/2: attention scores q
  float *DQ;                            // L(L-1)/2: their gradients
  float *G;                             // L × H: gradient of anchor_w1_l
  float *DU;                            // L × H: Σ_j of the pre-tanh attention gradients of layer l
  float *DA;                            // L × H: gradient reaching anchor l through later layers' inputs
  float *GW;                            // n_ops × H: gradient of w_emb (zeroed by the Adam pass)
  float *GG;                            // H: gradient of g_emb
  int *OPS, *SK, *NSK;                  // ops (L), skips (L(L-1)/2), skips per layer (L)
};

// ------------------------------------------------------------------------------------------------ small helpers
__device__ __forceinline__ float en_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float en_warp_max(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ int en_warp_min(int v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// block-wide reductions (every thread gets the result); red: EN_NW floats of shared memory
__device__ float en_block_max(float v, float* red) {
  v = en_warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = (threadIdx.x & 31) < EN_NW ? red[threadIdx.x & 31] : -INFINITY;
  return en_warp_max(r);
}
__device__ int en_block_min(int v, int* red) {
  v = en_warp_min(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  int r = (threadIdx.x & 31) < EN_NW ? red[threadIdx.x & 31] : 0x7fffffff;
  return en_warp_min(r);
}
__device__ __forceinline__ float en_sigmoid(float z) { return 1.f / (1.f + expf(-z)); }
// logit shaping s(z) = tanh_const · tanh(z / temperature), each factor skipped when its setting is None
__device__ __forceinline__ float en_shape(const EnCfg& cf, float z) {
  if (cf.use_temp) z = z / cf.temp;
  if (cf.use_tanh) z = cf.tanh_c * tanhf(z);
  return z;
}
__device__ __forceinline__ float en_dshape(const EnCfg& cf, float z) {
  float d = 1.f;
  if (cf.use_temp) {
    z = z / cf.temp;
    d = 1.f / cf.temp;
  }
  if (cf.use_tanh) {
    const float t = tanhf(z);
    d *= cf.tanh_c * (1.f - t * t);
  }
  return d;
}
__device__ __forceinline__ float en_uniform(const EnCfg& cf, long long draw, int arc, int dec) {
  uint32_t o[4];
  philox4x32_10((uint32_t)draw, (uint32_t)((unsigned long long)draw >> 32), (uint32_t)arc, (uint32_t)dec, cf.k0, cf.k1, o);
  return (float)(o[0] >> 8) * 5.9604644775390625e-8f;
}

// y[b·ldy + j] = Σ_k x[b·ldx + k] · W[k·ldw + j] for j < N, b < B (k in order): each weight is read once for the B arcs
template <int B>
__device__ __forceinline__ void en_mv_rows(const float* W, int ldw, const float* x, int ldx, int K, int N, float* y, int ldy) {
  for (int j = threadIdx.x; j < N; j += EN_NT) {
    float acc[B];
#pragma unroll
    for (int b = 0; b < B; b++) acc[b] = 0.f;
    for (int k = 0; k < K; k++) {
      const float w = W[(size_t)k * ldw + j];
#pragma unroll
      for (int b = 0; b < B; b++) acc[b] = fmaf(x[b * ldx + k], w, acc[b]);
    }
#pragma unroll
    for (int b = 0; b < B; b++) y[b * ldy + j] = acc[b];
  }
}
// y[k] = Σ_j W[k·ldw + j] · d[j] for k < K: one warp per row, lanes strided over j, then an xor-butterfly sum
__device__ __forceinline__ void en_mv_cols(const float* W, int ldw, const float* d, int K, int N, float* y) {
  const int lane = threadIdx.x & 31;
  for (int k = threadIdx.x >> 5; k < K; k += EN_NW) {
    float acc = 0.f;
    for (int j = lane; j < N; j += 32) acc = fmaf(W[(size_t)k * ldw + j], d[j], acc);
    acc = en_warp_sum(acc);
    if (lane == 0) y[k] = acc;
  }
}

// Draw from the categorical of weights e[0..n) (already exp(s - max)): the first i whose inclusive prefix sum exceeds
// u·total.  Every thread takes a contiguous chunk; chunk sums are scanned warp by warp and then across warps in a fixed
// order.  Returns the index (all threads) and the total in *total_out (all threads).  red: 4·EN_NW + 1 words (warp
// totals, warp offsets, the total, the block minimum's scratch).
__device__ int en_draw(const float* e, int n, float u, float* total_out, float* red) {
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int chunk = (n + EN_NT - 1) / EN_NT;
  const int i0 = min(tid * chunk, n), i1 = min(i0 + chunk, n);
  float s = 0.f;
  for (int i = i0; i < i1; i++) s += e[i];
  float inc = s;                                            // warp inclusive scan (fixed shfl_up tree)
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  __syncthreads();
  if (lane == 31) red[w] = inc;
  __syncthreads();
  if (tid == 0) {                                           // warp offsets, in warp order
    float run = 0.f;
    for (int q = 0; q < EN_NW; q++) {
      const float t = red[q];
      red[EN_NW + q] = run;
      run += t;
    }
    red[2 * EN_NW] = run;
  }
  __syncthreads();
  const float total = red[2 * EN_NW];
  float run = red[EN_NW + w] + inc - s;                     // exclusive prefix of this thread's chunk
  const float thr = u * total;
  int pick = 0x7fffffff;
  for (int i = i0; i < i1; i++) {
    run += e[i];
    if (thr < run) {
      pick = i;
      break;
    }
  }
  pick = en_block_min(pick, (int*)red + 3 * EN_NW);
  if (pick == 0x7fffffff) {                                 // u·total reached the total by rounding: the last bin with weight
    int last = -1;
    for (int i = tid; i < n; i += EN_NT)
      if (e[i] > 0.f) last = i;
    pick = -en_block_min(-last, (int*)red + 3 * EN_NW);     // the maximum index, as a minimum of negatives
    if (pick < 0) pick = n - 1;                             // unreachable: the bin of the maximum has weight 1
  }
  *total_out = total;
  return pick;
}

// ------------------------------------------------------------------------------------------------ the sampler
// Shared memory of en_forward (floats unless noted): xh B×2H, c B×H, gt B×4H, z B×n_ops, hw2 B×H, per-arc accumulators
// B×8, per-(arc, anchor) decision records B×L×4, int skips B×L, reduction scratch 6·EN_NW.
struct EnSmem {
  float *xh, *c, *gt, *z, *hw2, *red, *acc, *rec;
  int* sk;
};
__host__ __device__ inline size_t en_smem_bytes(int B, int L, int H, int n_ops) {
  return 4 * ((size_t)B * (2 * H + H + 4 * H + n_ops + H + 8 + 4 * L + L) + 6 * EN_NW);
}
__device__ inline EnSmem en_carve(float* base, int B, int L, int H, int n_ops) {
  EnSmem m;
  m.xh = base;
  m.c = m.xh + B * 2 * H;
  m.gt = m.c + B * H;
  m.z = m.gt + B * 4 * H;
  m.hw2 = m.z + (size_t)B * n_ops;
  m.acc = m.hw2 + B * H;
  m.rec = m.acc + B * 8;
  m.sk = (int*)(m.rec + B * 4 * L);
  m.red = (float*)(m.sk + B * L);
  return m;
}

// One LSTM cell for B arcs: gates = [x, h]·w_lstm, then c, h in place.  TRAIN saves [x, h_prev], c_prev, the gates and
// the new c into the cell's rows of the scratch (n = cell index).
template <int B, bool TRAIN>
__device__ void en_cell(const EnCfg& cf, const float* P, EnSmem& sm, const EnBufs& bf, int n) {
  const int H = cf.H;
  en_mv_rows<B>(P + cf.o_lstm, 4 * H, sm.xh, 2 * H, 2 * H, 4 * H, sm.gt, 4 * H);
  __syncthreads();
  for (int idx = threadIdx.x; idx < B * H; idx += EN_NT) {
    const int b = idx / H, k = idx - b * H;
    float* g = sm.gt + b * 4 * H;
    const float i = en_sigmoid(g[k]), f = en_sigmoid(g[H + k]), o = en_sigmoid(g[2 * H + k]), gg = tanhf(g[3 * H + k]);
    const float cp = sm.c[b * H + k];
    const float cn = fmaf(i, gg, f * cp);
    const float hn = o * tanhf(cn);
    if (TRAIN) {
      bf.XH[(size_t)n * 2 * H + k] = sm.xh[k];
      bf.XH[(size_t)n * 2 * H + H + k] = sm.xh[H + k];
      bf.CS[(size_t)n * H + k] = cp;
      float* gt = bf.GT + (size_t)n * 4 * H;
      gt[k] = i;
      gt[H + k] = f;
      gt[2 * H + k] = o;
      gt[3 * H + k] = gg;
    }
    sm.c[b * H + k] = cn;
    sm.xh[b * 2 * H + H + k] = hn;
  }
  __syncthreads();
}

// The sampler for B arcs (arc ids arc0 .. arc0 + B - 1; those >= n_arcs are computed and discarded).  TRAIN (B = 1):
// decisions may be imposed (arc_in), and everything the backward pass needs is saved; acc[0..3] of arc 0 receive
// nll, ent, Σ_l kl_l and the number of skips.  Sampling: uniforms may be imposed; probabilities may be written out.
template <int B, bool TRAIN>
__device__ void en_forward(const EnCfg& cf, const float* P, EnSmem& sm, const EnBufs& bf, float* ANC, float* AW1, int arc0, int n_arcs,
                           long long draw, const int* arc_in, const float* u_in, int* arcs_out, float* op_probs, float* skip_probs) {
  const int H = cf.H, L = cf.L, n_ops = cf.n_ops, tid = threadIdx.x;
  const float* g_emb = P + cf.o_gemb;
  for (int idx = tid; idx < B * H; idx += EN_NT) {
    const int b = idx / H, k = idx - b * H;
    sm.xh[b * 2 * H + k] = g_emb[k];
    sm.xh[b * 2 * H + H + k] = 0.f;
    sm.c[b * H + k] = 0.f;
  }
  if (tid < B * 8) sm.acc[tid] = 0.f;
  __syncthreads();
  for (int l = 0; l < L; l++) {
    const int pos = l * (l + 1) / 2;            // this layer's first decision in the arc
    // ---- cell A, then the op decision
    en_cell<B, TRAIN>(cf, P, sm, bf, 2 * l);
    en_mv_rows<B>(P + cf.o_soft, n_ops, sm.xh + H, 2 * H, H, n_ops, sm.z, n_ops);
    __syncthreads();
    for (int b = 0; b < B; b++) {
      float* z = sm.z + (size_t)b * n_ops;
      float mx = -INFINITY;
      for (int i = tid; i < n_ops; i += EN_NT) {
        const float s = en_shape(cf, z[i]);
        if (TRAIN) bf.Z[(size_t)l * n_ops + i] = z[i];
        z[i] = s;
        mx = fmaxf(mx, s);
      }
      mx = en_block_max(mx, sm.red);
      for (int i = tid; i < n_ops; i += EN_NT) z[i] = expf(z[i] - mx);
      __syncthreads();
      const int arc = arc0 + b;
      float u = 0.f;
      if (!(TRAIN && arc_in)) u = u_in ? (arc < n_arcs ? u_in[(size_t)arc * cf.A + pos] : 0.f) : en_uniform(cf, draw, arc, pos);
      float total;
      int op = en_draw(z, n_ops, u, &total, sm.red + EN_NW);
      if (TRAIN && arc_in) op = arc_in[pos];
      if (TRAIN || op_probs) {
        for (int i = tid; i < n_ops; i += EN_NT) {
          const float p = z[i] / total;
          if (TRAIN) bf.PR[(size_t)l * n_ops + i] = p;
          else if (arc < n_arcs) op_probs[((size_t)arc * L + l) * n_ops + i] = p;
        }
      }
      if (tid == 0) {
        if (TRAIN) {
          const float ce = logf(total) + mx - en_shape(cf, bf.Z[(size_t)l * n_ops + op]);
          sm.acc[0] += ce;
          sm.acc[1] += ce * expf(-ce);
          bf.OPS[l] = op;
        }
        if (arcs_out && arc < n_arcs) arcs_out[(size_t)arc * cf.A + pos] = op;
        sm.sk[b * L + 0] = op;                  // parked until the embedding row is loaded below
      }
      __syncthreads();
    }
    const float* w_emb = P + cf.o_wemb;
    for (int idx = tid; idx < B * H; idx += EN_NT) {
      const int b = idx / H, k = idx - b * H;
      sm.xh[b * 2 * H + k] = w_emb[(size_t)sm.sk[b * L] * H + k];
    }
    __syncthreads();
    // ---- cell B, then the skip decisions against the anchors of layers j < l
    en_cell<B, TRAIN>(cf, P, sm, bf, 2 * l + 1);
    if (l > 0) {
      en_mv_rows<B>(P + cf.o_w2, H, sm.xh + H, 2 * H, H, H, sm.hw2, H);
      __syncthreads();
      const float* v = P + cf.o_v;
      const int base = l * (l - 1) / 2;
      for (int bj = tid >> 5; bj < B * l; bj += EN_NW) {    // one warp per (arc, anchor)
        const int b = bj / l, j = bj - b * l, lane = tid & 31, arc = arc0 + b;
        const float* aw = AW1 + ((size_t)b * L + j) * H;
        float q = 0.f;
        for (int k = lane; k < H; k += 32) {
          const float t = tanhf(aw[k] + sm.hw2[b * H + k]);
          if (TRAIN) bf.TA[(size_t)(base + j) * H + k] = t;
          q = fmaf(t, v[k], q);
        }
        q = en_warp_sum(q);
        if (lane == 0) {
          const float s0 = en_shape(cf, -q), s1 = en_shape(cf, q), mx = fmaxf(s0, s1);
          const float e0 = expf(s0 - mx), e1 = expf(s1 - mx), tot = e0 + e1;
          int skip;
          if (TRAIN && arc_in) skip = arc_in[pos + 1 + j];
          else {
            const float u = u_in ? (arc < n_arcs ? u_in[(size_t)arc * cf.A + pos + 1 + j] : 0.f) : en_uniform(cf, draw, arc, pos + 1 + j);
            skip = u * tot < e0 ? 0 : 1;
          }
          float* r = sm.rec + ((size_t)b * L + j) * 4;
          if (TRAIN) {
            const float ce = logf(tot) + mx - (skip ? s1 : s0);
            const float g0 = en_sigmoid(s0), g1 = en_sigmoid(s1);
            r[0] = ce;
            r[1] = ce * expf(-ce);
            r[2] = g0 * logf(g0 / (1.f - cf.skip_target)) + g1 * logf(g1 / cf.skip_target);
            bf.Q[base + j] = q;
            bf.SK[base + j] = skip;
          }
          if (skip_probs && arc < n_arcs) skip_probs[(size_t)arc * (L * (L - 1) / 2) + base + j] = e1 / tot;
          if (arcs_out && arc < n_arcs) arcs_out[(size_t)arc * cf.A + pos + 1 + j] = skip;
          sm.sk[b * L + j] = skip;
        }
      }
      __syncthreads();
      if (tid < B) {                            // per-arc sums over the anchors, in anchor order
        float* a = sm.acc + tid * 8;
        float kl = 0.f;
        int ns = 0;
        for (int j = 0; j < l; j++) {
          const float* r = sm.rec + ((size_t)tid * L + j) * 4;
          if (TRAIN) {
            a[0] += r[0];
            a[1] += r[1];
            kl += r[2];
          }
          ns += sm.sk[tid * L + j];
        }
        a[2] += kl;
        a[3] += (float)ns;
        a[4] = (float)ns;
        if (TRAIN) bf.NSK[l] = ns;
      }
      __syncthreads();
      for (int idx = tid; idx < B * H; idx += EN_NT) {      // next input: the mean of the chosen anchors (and 1 for none)
        const int b = idx / H, k = idx - b * H;
        float s = 0.f;
        for (int j = 0; j < l; j++)
          if (sm.sk[b * L + j]) s += ANC[((size_t)b * L + j) * H + k];
        sm.xh[b * 2 * H + k] = s / (1.f + sm.acc[b * 8 + 4]);
      }
    } else {
      if (TRAIN && tid == 0) bf.NSK[0] = 0;
      for (int idx = tid; idx < B * H; idx += EN_NT) {
        const int b = idx / H, k = idx - b * H;
        sm.xh[b * 2 * H + k] = g_emb[k];
      }
    }
    // ---- append the anchor h and anchor·w_attn_1 (the new input lives in xh[0:H] and is not touched here)
    for (int idx = tid; idx < B * H; idx += EN_NT) {
      const int b = idx / H, k = idx - b * H;
      ANC[((size_t)b * L + l) * H + k] = sm.xh[b * 2 * H + H + k];
    }
    en_mv_rows<B>(P + cf.o_w1, H, sm.xh + H, 2 * H, H, H, sm.hw2, H);
    __syncthreads();
    for (int idx = tid; idx < B * H; idx += EN_NT) {
      const int b = idx / H, k = idx - b * H;
      AW1[((size_t)b * L + l) * H + k] = sm.hw2[b * H + k];
    }
    __syncthreads();
  }
  if (TRAIN) {                                  // row 2L of XH: [0, h_final] and the final c
    for (int k = tid; k < H; k += EN_NT) {
      bf.XH[(size_t)2 * L * 2 * H + k] = 0.f;
      bf.XH[(size_t)2 * L * 2 * H + H + k] = sm.xh[H + k];
      bf.CS[(size_t)2 * L * H + k] = sm.c[k];
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ backward + Adam
// Backward through cell n: (dh, dc) of its outputs -> dz (shared, and DZS[n]), dc of its input c (in place), then
// dxh = w_lstm · dz (2H: dx, dh_prev).
__device__ void en_cell_bwd(const EnCfg& cf, const float* P, const EnBufs& bf, int n, const float* dh, float* dc, float* dz, float* dxh) {
  const int H = cf.H;
  for (int k = threadIdx.x; k < H; k += EN_NT) {
    const float* gt = bf.GT + (size_t)n * 4 * H;
    const float i = gt[k], f = gt[H + k], o = gt[2 * H + k], g = gt[3 * H + k];
    const float cp = bf.CS[(size_t)n * H + k], cn = bf.CS[(size_t)(n + 1) * H + k];
    const float tc = tanhf(cn);
    const float dct = dc[k] + dh[k] * o * (1.f - tc * tc);
    float* d = bf.DZS + (size_t)n * 4 * H;
    const float zi = dct * g * i * (1.f - i), zf = dct * cp * f * (1.f - f), zo = dh[k] * tc * o * (1.f - o), zg = dct * i * (1.f - g * g);
    dz[k] = d[k] = zi;
    dz[H + k] = d[H + k] = zf;
    dz[2 * H + k] = d[2 * H + k] = zo;
    dz[3 * H + k] = d[3 * H + k] = zg;
    dc[k] = dct * f;
  }
  __syncthreads();
  en_mv_cols(P + cf.o_lstm, 4 * H, dz, 2 * H, 4 * H, dxh);
  __syncthreads();
}

// Adam (TF, β1 = 0) on param[k·N + j] for k < K, j < N with gradient Σ_t X[t·ldx + k] · Y[t·ldy + j] (t in order).
// One work item = one column j and 8 consecutive rows.
__device__ void en_adam_outer(float* p, float* m, float* v, int K, int N, const float* X, int ldx, const float* Y, int ldy, int T, float lr_t) {
  const int kb = (K + 7) / 8;
  for (int it = threadIdx.x; it < kb * N; it += EN_NT) {
    const int j = it % N, k0 = (it / N) * 8;
    float acc[8];
#pragma unroll
    for (int q = 0; q < 8; q++) acc[q] = 0.f;
    for (int t = 0; t < T; t++) {
      const float y = Y[(size_t)t * ldy + j];
#pragma unroll
      for (int q = 0; q < 8; q++)
        if (k0 + q < K) acc[q] = fmaf(X[(size_t)t * ldx + k0 + q], y, acc[q]);
    }
#pragma unroll
    for (int q = 0; q < 8; q++) {
      if (k0 + q >= K) break;
      const size_t e = (size_t)(k0 + q) * N + j;
      const float g = acc[q];
      const float vv = 0.999f * v[e] + 0.001f * (g * g);
      v[e] = vv;
      m[e] = g;
      p[e] -= lr_t * g / (sqrtf(vv) + 1e-3f);
    }
  }
}
__device__ void en_adam_dense(float* p, float* m, float* v, float* g_in, int n, float lr_t, bool clear) {
  for (int e = threadIdx.x; e < n; e += EN_NT) {
    const float g = g_in[e];
    if (clear) g_in[e] = 0.f;
    const float vv = 0.999f * v[e] + 0.001f * (g * g);
    v[e] = vv;
    m[e] = g;
    p[e] -= lr_t * g / (sqrtf(vv) + 1e-3f);
  }
}

// b2p0 = β2^(Adam steps taken so far), from the host's copy of the step count
__global__ void __launch_bounds__(EN_NT) enas_train_kernel(EnCfg cf, float* P, float* Mo, float* Vo, EnDev* st, float R, int T,
                                                           const int* arcs_in, float* stats, EnBufs bf, double b2p0) {
  extern __shared__ float en_sm[];
  const int H = cf.H, L = cf.L, n_ops = cf.n_ops, tid = threadIdx.x;
  EnSmem sm = en_carve(en_sm, 1, L, H, n_ops);
  // backward work vectors reuse the sampler's shared memory: dh, dc, dhb, tmp (H each) in hw2.. and z; dz, dxh in gt, xh
  float* dz = sm.gt;                            // 4H
  float* dxh = sm.xh;                           // 2H
  float* zs = sm.z;                             // n_ops
  __shared__ float s_dh[EN_MAXH], s_dc[EN_MAXH], s_dhb[EN_MAXH], s_ta[EN_MAXH], s_tb[EN_MAXH];
  __shared__ float s_scal[4];
  __shared__ long long s_cnt[2];
  if (tid == 0) {
    s_scal[0] = st->baseline;
    s_cnt[0] = st->step;
    s_cnt[1] = st->draws;
    int bad = 0;
    for (int t = 0; arcs_in && t < T && !bad; t++)
      for (int l = 0; l < L; l++) {
        const int* a = arcs_in + (size_t)t * cf.A + l * (l + 1) / 2;
        if (a[0] < 0 || a[0] >= n_ops) bad = 1;
        for (int j = 0; j < l; j++)
          if (a[1 + j] != 0 && a[1 + j] != 1) bad = 1;
      }
    st->err = bad;
    s_scal[3] = (float)bad;
  }
  __syncthreads();
  if (s_scal[3] != 0.f) return;
  const int npairs = L * (L - 1) / 2;
  double b2p = b2p0;
  for (int step = 0; step < T; step++) {
    const long long draw = s_cnt[1] + step;
    en_forward<1, true>(cf, P, sm, bf, bf.ANC, bf.AW1, 0, 1, draw, arcs_in ? arcs_in + (size_t)step * cf.A : nullptr, nullptr, nullptr,
                        nullptr, nullptr);
    // ---- reward, baseline, loss (thread 0), broadcast the advantage
    if (tid == 0) {
      const float nll = sm.acc[0], ent = sm.acc[1], klsum = sm.acc[2], nskip = sm.acc[3];
      const float r = R + cf.ent_w * ent;
      float b = s_scal[0];
      b = b - (1.f - cf.decay) * (b - r);
      s_scal[0] = b;
      const float adv = r - b;
      const float klm = L > 1 ? klsum / (float)(L - 1) : 0.f;
      s_scal[1] = adv;
      s_scal[2] = L > 1 ? cf.skip_w / (float)(L - 1) : 0.f;
      if (stats) {
        float* o = stats + (size_t)step * EN_NSTAT;
        o[0] = nll;
        o[1] = ent;
        o[2] = klm;
        o[3] = nll * adv + cf.skip_w * klm;
        o[4] = b;
        o[5] = npairs ? nskip / (float)npairs : 0.f;
      }
    }
    for (int e = tid; e < L * H; e += EN_NT) bf.G[e] = bf.DA[e] = bf.DU[e] = 0.f;
    for (int k = tid; k < H; k += EN_NT) s_dh[k] = s_dc[k] = bf.GG[k] = 0.f;
    __syncthreads();
    const float adv = s_scal[1], skc = s_scal[2];
    const float t0 = 1.f - cf.skip_target, t1 = cf.skip_target;
    const float* W1 = P + cf.o_w1;
    const float* W2 = P + cf.o_w2;
    const float* v = P + cf.o_v;
    for (int l = L - 1; l >= 0; l--) {
      const int base = l * (l - 1) / 2;
      if (l > 0) {                              // skip decisions of layer l: CE and kl gradients -> dq -> du
        for (int j = tid >> 5; j < l; j += EN_NW) {
          if ((tid & 31) == 0) {
            const float q = bf.Q[base + j];
            const int skip = bf.SK[base + j];
            const float s0 = en_shape(cf, -q), s1 = en_shape(cf, q), mx = fmaxf(s0, s1);
            const float e0 = expf(s0 - mx), e1 = expf(s1 - mx), tot = e0 + e1;
            const float p0 = e0 / tot, p1 = e1 / tot;
            const float g0 = en_sigmoid(s0), g1 = en_sigmoid(s1);
            const float ds0 = adv * (p0 - (skip == 0 ? 1.f : 0.f)) + skc * g0 * (1.f - g0) * (logf(g0 / t0) + 1.f);
            const float ds1 = adv * (p1 - (skip == 1 ? 1.f : 0.f)) + skc * g1 * (1.f - g1) * (logf(g1 / t1) + 1.f);
            bf.DQ[base + j] = ds1 * en_dshape(cf, q) - ds0 * en_dshape(cf, -q);
          }
        }
        __syncthreads();
        for (int k = tid; k < H; k += EN_NT) {
          float su = 0.f;
          for (int j = 0; j < l; j++) {
            const float t = bf.TA[(size_t)(base + j) * H + k];
            const float du = bf.DQ[base + j] * v[k] * (1.f - t * t);
            su += du;
            bf.G[(size_t)j * H + k] += du;
          }
          bf.DU[(size_t)l * H + k] = su;
        }
        __syncthreads();
      }
      // gradient of h_B(l) = anchor l: recurrence + later inputs + its w_attn_1 row + this layer's w_attn_2 query
      en_mv_cols(W1, H, bf.G + (size_t)l * H, H, H, s_ta);
      if (l > 0) en_mv_cols(W2, H, bf.DU + (size_t)l * H, H, H, s_tb);
      __syncthreads();
      for (int k = tid; k < H; k += EN_NT) s_dhb[k] = s_dh[k] + bf.DA[(size_t)l * H + k] + s_ta[k] + (l > 0 ? s_tb[k] : 0.f);
      __syncthreads();
      en_cell_bwd(cf, P, bf, 2 * l + 1, s_dhb, s_dc, dz, dxh);
      const int op = bf.OPS[l];
      for (int k = tid; k < H; k += EN_NT) {
        bf.GW[(size_t)op * H + k] += dxh[k];
        s_dh[k] = dxh[H + k];
      }
      // op decision of layer l: CE gradient through the shaping -> dz_soft (kept in Z for w_soft's gradient)
      for (int i = tid; i < n_ops; i += EN_NT) {
        const size_t e = (size_t)l * n_ops + i;
        const float d = adv * (bf.PR[e] - (i == op ? 1.f : 0.f)) * en_dshape(cf, bf.Z[e]);
        zs[i] = d;
        bf.Z[e] = d;
      }
      __syncthreads();
      en_mv_cols(P + cf.o_soft, n_ops, zs, H, n_ops, s_ta);
      __syncthreads();
      for (int k = tid; k < H; k += EN_NT) s_dh[k] += s_ta[k];
      __syncthreads();
      en_cell_bwd(cf, P, bf, 2 * l, s_dh, s_dc, dz, dxh);
      for (int k = tid; k < H; k += EN_NT) {
        s_dh[k] = dxh[H + k];
        const float dx = dxh[k];
        if (l <= 1) bf.GG[k] += dx;             // the input of cell A(0) and A(1) is g_emb
        else {
          const int pb = (l - 1) * (l - 2) / 2;
          const float w = 1.f + (float)bf.NSK[l - 1];
          for (int j = 0; j < l - 1; j++)
            if (bf.SK[pb + j]) bf.DA[(size_t)j * H + k] += dx / w;
        }
      }
      __syncthreads();
    }
    // ---- weight gradients and Adam (β1 = 0, β2 = 0.999, ε̂ = 1e-3, lr_t = lr·sqrt(1 - β2^t))
    b2p *= 0.999;                               // β2^t, t = s_cnt[0] + step + 1, as a running product like TF's beta2_power
    const float lr_t = (float)((double)cf.lr * sqrt(1.0 - b2p));
    // w_lstm: Σ over cells of [x, h_prev] ⊗ dz; w_soft: Σ_l h_A(l) ⊗ dz_soft(l); w_attn_1 / w_attn_2: Σ_l anchor_l ⊗ G_l / DU_l
    // (anchor l = h after cell B(l) = row 2l + 2 of XH); v_attn: Σ over skip decisions of dq · tanh row
    en_adam_outer(P + cf.o_lstm, Mo + cf.o_lstm, Vo + cf.o_lstm, 2 * H, 4 * H, bf.XH, 2 * H, bf.DZS, 4 * H, 2 * L, lr_t);
    en_adam_outer(P + cf.o_soft, Mo + cf.o_soft, Vo + cf.o_soft, H, n_ops, bf.XH + 3 * H, 4 * H, bf.Z, n_ops, L, lr_t);
    en_adam_outer(P + cf.o_w1, Mo + cf.o_w1, Vo + cf.o_w1, H, H, bf.XH + 5 * H, 4 * H, bf.G, H, L, lr_t);
    en_adam_outer(P + cf.o_w2, Mo + cf.o_w2, Vo + cf.o_w2, H, H, bf.XH + 5 * H, 4 * H, bf.DU, H, L, lr_t);
    en_adam_outer(P + cf.o_v, Mo + cf.o_v, Vo + cf.o_v, 1, H, bf.DQ, 1, bf.TA, H, npairs, lr_t);
    en_adam_dense(P + cf.o_gemb, Mo + cf.o_gemb, Vo + cf.o_gemb, bf.GG, H, lr_t, false);
    en_adam_dense(P + cf.o_wemb, Mo + cf.o_wemb, Vo + cf.o_wemb, bf.GW, n_ops * H, lr_t, true);
    __syncthreads();
  }
  if (tid == 0) {
    st->baseline = s_scal[0];
    st->step = s_cnt[0] + T;
    st->draws = s_cnt[1] + T;
  }
}

__global__ void __launch_bounds__(EN_NT) enas_sample_kernel(EnCfg cf, const float* __restrict__ P, const EnDev* __restrict__ st, int n_arcs,
                                                            const float* __restrict__ u_in, int* __restrict__ arcs_out, float* __restrict__ op_probs,
                                                            float* __restrict__ skip_probs, float* __restrict__ scratch) {
  extern __shared__ float en_sm[];
  EnSmem sm = en_carve(en_sm, EN_SB, cf.L, cf.H, cf.n_ops);
  float* ANC = scratch + (size_t)blockIdx.x * 2 * EN_SB * cf.L * cf.H;
  float* AW1 = ANC + (size_t)EN_SB * cf.L * cf.H;
  const EnBufs none{};
  en_forward<EN_SB, false>(cf, P, sm, none, ANC, AW1, blockIdx.x * EN_SB, n_arcs, st->draws, nullptr, u_in, arcs_out, op_probs, skip_probs);
}

__global__ void enas_bump_kernel(EnDev* st) { st->draws += 1; }

// U(-0.1, 0.1) initial parameters: element i takes word 0 of Philox counter (i lo, i hi, 2^32 - 1, 2^32 - 1), a counter no
// draw uses (draws have arc < 2^32 - 1)
__global__ void enas_init_kernel(float* P, long long n, uint32_t k0, uint32_t k1) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    uint32_t o[4];
    philox4x32_10((uint32_t)i, (uint32_t)((unsigned long long)i >> 32), 0xFFFFFFFFu, 0xFFFFFFFFu, k0, k1, o);
    P[i] = (float)(o[0] >> 8) * 5.9604644775390625e-8f * 0.2f - 0.1f;
  }
}

// ------------------------------------------------------------------------------------------------ host side
struct kbo_enas {
  EnCfg cf{};
  DevBuf<float> par, mom, var, sscr;
  DevBuf<float> scr;   // the training kernel's float arrays, then its int arrays OPS / SK / NSK (en_carve_scratch): both types
  DevBuf<EnDev> dev;
  EnBufs bf{};
  EventSet<4> ev;
  float last_ms[2] = {};
  long long step = 0;                   // host copy of the Adam step count (the kernel's β2^t starts from it)
};

static int en_carve_scratch(kbo_handle* h, kbo_enas* e, cudaStream_t s) {
  const size_t L = e->cf.L, H = e->cf.H, n = e->cf.n_ops, np = L * (L - 1) / 2;
  const size_t nf[] = {(2 * L + 1) * 2 * H, (2 * L + 1) * H, 2 * L * 4 * H, 2 * L * 4 * H, L * n, L * n, L * H, L * H,
                       np * H, np, np, L * H, L * H, L * H, n * H, H};
  size_t total = 0;
  for (size_t f : nf) total += (f + 31) / 32 * 32;
  const size_t ints = L + np + L + 3;
  KBO_TRY(kbo_reserve(h, e->scr, total + ints));
  KBO_CUDA(h, cudaMemsetAsync(e->scr.p, 0, sizeof *e->scr.p * (total + ints), s));
  float* p = e->scr.p;
  float** dst[] = {&e->bf.XH, &e->bf.CS, &e->bf.GT, &e->bf.DZS, &e->bf.Z, &e->bf.PR, &e->bf.ANC, &e->bf.AW1,
                   &e->bf.TA, &e->bf.Q, &e->bf.DQ, &e->bf.G, &e->bf.DU, &e->bf.DA, &e->bf.GW, &e->bf.GG};
  for (int i = 0; i < 16; i++) {
    *dst[i] = p;
    p += (nf[i] + 31) / 32 * 32;
  }
  int* q = reinterpret_cast<int*>(p);   // ints after the floats: same size, and every float array starts 128-byte aligned
  e->bf.OPS = q;
  e->bf.SK = q + L;
  e->bf.NSK = q + L + np + 1;
  return KBO_OK;
}

// The controller's buffers, events and initial parameters (uniform in [-0.1, 0.1)), with the work queued on cs.
static int en_setup(kbo_handle* h, kbo_enas* e, cudaStream_t cs) {
  const long long o = e->cf.n_par;
  KBO_TRY(kbo_reserve(h, e->par, (size_t)o));
  KBO_TRY(kbo_reserve(h, e->mom, (size_t)o));
  KBO_TRY(kbo_reserve(h, e->var, (size_t)o));
  KBO_TRY(kbo_reserve(h, e->dev, 1));
  KBO_TRY(en_carve_scratch(h, e, cs));
  KBO_TRY(e->ev.create());
  const EnDev d0{0.f, 0, 0, 0};
  KBO_CUDA(h, cudaMemsetAsync(e->mom.p, 0, sizeof *e->mom.p * (size_t)o, cs));
  KBO_CUDA(h, cudaMemsetAsync(e->var.p, 0, sizeof *e->var.p * (size_t)o, cs));
  KBO_CUDA(h, kbo_copy(e->dev.p, &d0, 1, cudaMemcpyHostToDevice, cs));
  enas_init_kernel<<<(int)std::min<long long>((o + 255) / 256, 1024), 256, 0, cs>>>(e->par.p, o, e->cf.k0, e->cf.k1);
  KBO_CUDA(h, cudaGetLastError());
  return KBO_OK;
}

extern "C" {

int kbo_enas_create(kbo_handle* h, kbo_enas** out, int32_t L, int32_t H, int32_t n_ops, const kbo_enas_settings* s, uint64_t seed) {
  if (!h || !out || !s) return KBO_ERR_INVALID;
  *out = nullptr;
  if (L < 1 || L > EN_MAXL) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_enas_create: 1 <= num_layers <= %d supported (got %d)", EN_MAXL, L);
  if (H < 1 || H > EN_MAXH) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_enas_create: 1 <= controller_hidden_size <= %d supported (got %d)", EN_MAXH, H);
  if (n_ops < 1 || n_ops > EN_MAXOPS) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_enas_create: 1 <= n_ops <= %d supported (got %d)", EN_MAXOPS, n_ops);
  if (!(s->baseline_decay >= 0.0 && s->baseline_decay <= 1.0)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_enas_create: baseline_decay must be in [0, 1]");
  if (!(s->learning_rate > 0.0 && s->learning_rate <= 1.0)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_enas_create: learning_rate must be in (0, 1]");
  if (!(s->skip_target > 0.0 && s->skip_target < 1.0)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_enas_create: skip_target must be in (0, 1)");
  if (!(s->entropy_weight >= 0.0) || !(s->skip_weight >= 0.0) || !std::isfinite(s->temperature) || !std::isfinite(s->tanh_const))
    KBO_FAIL(h, KBO_ERR_INVALID, "kbo_enas_create: entropy_weight and skip_weight must be >= 0, temperature and tanh_const finite");
  KBO_CUDA(h, cudaSetDevice(h->device));
  std::unique_ptr<kbo_enas> e(new (std::nothrow) kbo_enas());
  if (!e) return KBO_ERR_NOMEM;
  EnCfg& c = e->cf;
  c.L = L;
  c.H = H;
  c.n_ops = n_ops;
  c.A = L * (L + 1) / 2;
  c.use_temp = s->temperature > 0.0;
  c.temp = c.use_temp ? (float)s->temperature : 1.f;
  c.use_tanh = s->tanh_const > 0.0;
  c.tanh_c = c.use_tanh ? (float)s->tanh_const : 1.f;
  c.ent_w = (float)s->entropy_weight;
  c.decay = (float)s->baseline_decay;
  c.lr = (float)s->learning_rate;
  c.skip_target = (float)s->skip_target;
  c.skip_w = (float)s->skip_weight;
  c.k0 = (uint32_t)seed;
  c.k1 = (uint32_t)(seed >> 32);
  long long o = 0;
  c.o_lstm = o; o += 8LL * H * H;
  c.o_gemb = o; o += H;
  c.o_wemb = o; o += (long long)n_ops * H;
  c.o_soft = o; o += (long long)H * n_ops;
  c.o_w1 = o; o += (long long)H * H;
  c.o_w2 = o; o += (long long)H * H;
  c.o_v = o; o += H;
  c.n_par = o;
  // set-up work runs on a private non-blocking stream, so creating a controller never waits on (or stalls) other work
  // on the device
  cudaStream_t cs = nullptr;
  int r = cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking) == cudaSuccess ? en_setup(h, e.get(), cs) : KBO_ERR_CUDA;
  if (cs) {
    if (cudaStreamSynchronize(cs) != cudaSuccess && r == KBO_OK) r = KBO_ERR_CUDA;
    cudaStreamDestroy(cs);
  }
  // The dynamic shared-memory limit is an attribute of the kernel, shared by every controller in the process: it is set
  // to what the largest shape the engine accepts needs, never to this controller's own need.  Every create sets the same
  // values, so a controller made later (or on another thread) can never lower the limit under a live larger one.
  if (r == KBO_OK && (cudaFuncSetAttribute(enas_train_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)en_smem_bytes(1, EN_MAXL, EN_MAXH, EN_MAXOPS)) != cudaSuccess ||
                      cudaFuncSetAttribute(enas_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)en_smem_bytes(EN_SB, EN_MAXL, EN_MAXH, EN_MAXOPS)) != cudaSuccess))
    r = KBO_ERR_CUDA;
  if (r == KBO_ERR_CUDA) KBO_FAIL(h, r, "kbo_enas_create: CUDA setup failed");
  KBO_TRY(r);
  *out = e.release();
  return KBO_OK;
}

void kbo_enas_destroy(kbo_enas* e) {
  if (e) delete e;
}

int kbo_enas_train(kbo_handle* h, kbo_enas* e, double reward, int32_t steps, const int32_t* arcs, float* stats, void* stream) {
  if (!h || !e) return KBO_ERR_INVALID;
  if (steps < 0 || steps > EN_MAXT) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_enas_train: 0 <= steps <= %d supported (got %d)", EN_MAXT, steps);
  if (!std::isfinite(reward)) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_enas_train: the reward must be finite");
  if (steps == 0) return KBO_OK;
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  cudaEventRecord(e->ev[0], s);
  enas_train_kernel<<<1, EN_NT, en_smem_bytes(1, e->cf.L, e->cf.H, e->cf.n_ops), s>>>(e->cf, e->par.p, e->mom.p, e->var.p,
                                                                                   e->dev.p, (float)reward, steps, arcs, stats, e->bf,
                                                                                   std::pow(0.999, (double)e->step));
  KBO_LAUNCH_CHECK(h);
  cudaEventRecord(e->ev[1], s);
  int err = 0;
  KBO_CUDA(h, kbo_copy(&err, &e->dev.p->err, 1, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  cudaEventElapsedTime(&e->last_ms[0], e->ev[0], e->ev[1]);
  if (err) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_enas_train: an imposed arc has an op outside [0, n_ops) or a skip other than 0 / 1 (nothing was trained)");
  e->step += steps;
  return KBO_OK;
}

int kbo_enas_sample(kbo_handle* h, kbo_enas* e, int32_t k, int32_t* arcs, const float* uniforms, float* op_probs, float* skip_probs, void* stream) {
  if (!h || !e) return KBO_ERR_INVALID;
  if (!arcs) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_enas_sample: null output");
  if (k < 1 || k > EN_MAXK) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_enas_sample: 1 <= k <= %d supported (got %d)", EN_MAXK, k);
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  const int blocks = (k + EN_SB - 1) / EN_SB;
  KBO_TRY(kbo_reserve(h, e->sscr, (size_t)blocks * 2 * EN_SB * e->cf.L * e->cf.H));
  cudaEventRecord(e->ev[2], s);
  enas_sample_kernel<<<blocks, EN_NT, en_smem_bytes(EN_SB, e->cf.L, e->cf.H, e->cf.n_ops), s>>>(e->cf, e->par.p, e->dev.p, k,
                                                                                              uniforms, arcs, op_probs, skip_probs, e->sscr.p);
  KBO_LAUNCH_CHECK(h);
  enas_bump_kernel<<<1, 1, 0, s>>>(e->dev.p);
  KBO_LAUNCH_CHECK(h);
  cudaEventRecord(e->ev[3], s);
  KBO_CUDA(h, cudaStreamSynchronize(s));
  cudaEventElapsedTime(&e->last_ms[1], e->ev[2], e->ev[3]);
  return KBO_OK;
}

int kbo_enas_state(kbo_handle* h, kbo_enas* e, float* params, float* m, float* v, float* baseline, int64_t* step, int64_t* draws, void* stream) {
  if (!h || !e) return KBO_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  const size_t n = e->cf.n_par;
  EnDev d{};
  KBO_CUDA(h, kbo_d2h(params, e->par.p, n, s));
  KBO_CUDA(h, kbo_d2h(m, e->mom.p, n, s));
  KBO_CUDA(h, kbo_d2h(v, e->var.p, n, s));
  KBO_CUDA(h, kbo_copy(&d, e->dev.p, 1, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  if (baseline) *baseline = d.baseline;
  if (step) *step = d.step;
  if (draws) *draws = d.draws;
  return KBO_OK;
}

int kbo_enas_set_params(kbo_handle* h, kbo_enas* e, const float* params, const float* m, const float* v, float baseline, int64_t step, void* stream) {
  if (!h || !e) return KBO_ERR_INVALID;
  if (!params) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_enas_set_params: null params");
  if (step < 0) KBO_FAIL(h, KBO_ERR_INVALID, "kbo_enas_set_params: step must be >= 0");
  cudaStream_t s = (cudaStream_t)stream;
  KBO_CUDA(h, cudaSetDevice(h->device));
  const size_t n = e->cf.n_par;
  EnDev d{};
  KBO_CUDA(h, kbo_copy(&d, e->dev.p, 1, cudaMemcpyDeviceToHost, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  d.baseline = baseline;
  d.step = step;
  KBO_CUDA(h, kbo_copy(e->par.p, params, n, cudaMemcpyHostToDevice, s));
  if (m) KBO_CUDA(h, kbo_copy(e->mom.p, m, n, cudaMemcpyHostToDevice, s));
  else KBO_CUDA(h, cudaMemsetAsync(e->mom.p, 0, sizeof *e->mom.p * n, s));
  if (v) KBO_CUDA(h, kbo_copy(e->var.p, v, n, cudaMemcpyHostToDevice, s));
  else KBO_CUDA(h, cudaMemsetAsync(e->var.p, 0, sizeof *e->var.p * n, s));
  KBO_CUDA(h, kbo_copy(e->dev.p, &d, 1, cudaMemcpyHostToDevice, s));
  KBO_CUDA(h, cudaStreamSynchronize(s));
  e->step = step;
  return KBO_OK;
}

int kbo_enas_last_timings(kbo_handle* h, kbo_enas* e, float* ms, int32_t n) {
  if (!h || !e) return KBO_ERR_INVALID;
  for (int i = 0; ms && i < n && i < 2; i++) ms[i] = e->last_ms[i];
  return 2;
}

}  // extern "C"
