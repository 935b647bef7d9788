// K* = amp·k(Xc, X) on the tensor cores, for the RANKING pass of the sweep ($SK/_gpr.py:446, $SK/kernels.py:1559-1570 RBF,
// :1713-1729 Matérn-5/2).  sm_90a: wgmma + TMA + mbarrier.
//
// The FP64 cross kernel (sweep.cu) spends ~75 FP64 operations per (candidate, trial) pair, on a
// pass whose output the ranking pass then rounds to fp16.  Here the pairwise distances are the dense product they are:
//     d²(c, x) = |c|² + |x|² − 2 c·x ,   c·x = Σ_d ĉ_d x̂_d   (ĉ, x̂: coordinates / ℓ_d, centred on the trials' mean, pre-scaled
//                                                              by √5 (Matérn) or 1/√2 (RBF) so the epilogue needs no constant)
// with c·x on the tensor cores.  Coordinates are split into fp16 hi + lo (|x̂ − hi − lo| ≤ 2⁻²²|x̂|) and all four partial
// products are accumulated in fp32 (small ones first), so c·x carries ~1e-7 relative error — the kernel value is then
// evaluated in fp32 (MUFU sqrt / ex2) per element by the epilogue warps, written ONCE as the fp16 hi plane the ranking kernel
// consumes (no lo plane, no FP64), and the normalised mean μ̃ = Σ_n K̃*[m,n]·alpha[n] is accumulated on the fly (four fp32 FMA
// chains, two per row, summed and added in FP64 once per 128-trial tile).  Both μ̃ and the variance built from this plane are only used to RANK: their error
// is measured per sweep on stratified calibration rows against the FP64 path and every candidate that could still be the
// maximum is re-evaluated in FP64 (sweep.cu).
//
// CTA = 128 candidate rows; it walks all 128-trial tiles.  Candidate planes (128 × Dp, hi and lo) stay in shared memory; trial
// planes stream through a 4-stage TMA ring one 32-feature slab at a time (SWIZZLE_64B), and each tile's (|x̂|², alpha) pairs (1 KB)
// arrive on the same barrier as its first slab, in a ring of their own, so the epilogue reads them with LDS;
//   warps 0-7  two consumer warpgroups (rows 64·wg …): per (tile, slab) 2 k-steps × 4 products of wgmma m64n128k16 into 64 fp32
//              registers, then the epilogue on those registers: d² → kernel → fp16 K* plane; μ̃ partials
//   warp 8     TMA producer
// The epilogue (~12 instructions and 2 MUFU per element) is the limiter; the MMAs take a fraction of that.  Tiles a pruning pass
// does not store run a body without the conversions, addresses and stores.
#include "kbo_internal.cuh"
#include <type_traits>

#include "tc_common.cuh"

#define KS_BM 128
#define KS_BN 128
#define KS_BK 32
#define KS_STAGES 4
#define KS_CONSUMERS 256                        // two warpgroups
#define KS_THREADS (KS_CONSUMERS + 32)
#define KS_A_PLANE_BYTES (KS_BM * KS_BK * 2)    // 8 KB: one plane of one slab of the candidate tile
#define KS_B_PLANE_BYTES (KS_BN * KS_BK * 2)    // 8 KB
#define KS_STAGE_BYTES (2 * KS_B_PLANE_BYTES)   // hi + lo
#define KS_MAX_SLABS 4                          // D <= 128
#define KS_NX_BYTES (KS_BN * 8)                 // 1 KB: one tile's (|x̂|², alpha) pairs, loaded with its first slab

namespace {
using namespace tcx;

struct KsSmem {
  uint64_t full[KS_STAGES];
  uint64_t empty[KS_STAGES];
  uint64_t a_full;
};

static size_t ks_smem_bytes(int ns) {
  return 1024 + (size_t)ns * 2 * KS_A_PLANE_BYTES + (size_t)KS_STAGES * (KS_STAGE_BYTES + KS_NX_BYTES) + 256;
}

__device__ __forceinline__ float ex2_ftz(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float sqrt_abs_ftz(float x) {   // MUFU.SQRT |x|: one instruction where max + rsqrt + multiply were three
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(fabsf(x)));
  return r;
}
// kernel value from the dot product: KIND 0 = RBF (coordinates pre-scaled by 1/√2: k = exp(−d2)), 1 = Matérn-5/2 (pre-scaled by
// √5: s = √d2, k = (1 + s + s²/3)·exp(−s)).  log2amp folds the amplitude into the exponent.
template <int KIND>
__device__ __forceinline__ float ks_kernel_value(float dot, float nsum, float log2amp) {
  float d2 = fmaf(-2.f, dot, nsum);
  if (KIND == 0) {
    d2 = fmaxf(d2, 0.f);
    return ex2_ftz(fmaf(d2, -1.4426950408889634f, log2amp));
  }
  const float s = sqrt_abs_ftz(d2);   // d2 < 0 only by rounding (|d2| tiny): its magnitude is as good an estimate as 0
  const float p = fmaf(fmaf(s, 0.33333334f, 1.f), s, 1.f);
  return p * ex2_ftz(fmaf(s, -1.4426950408889634f, log2amp));
}

template <int KIND>
__global__ void __launch_bounds__(KS_THREADS, 1)
tc_kstar_kernel(const __grid_constant__ CUtensorMap tmCh, const __grid_constant__ CUtensorMap tmCl, const __grid_constant__ CUtensorMap tmXh,
                const __grid_constant__ CUtensorMap tmXl, int ns, int ntiles, int N, const float* __restrict__ ncand,
                const float4* __restrict__ nxal4 /* (|x̂_n|², alpha_n) pairs, two trials per float4 */, int nx_tiles /* tiles that have pairs */,
                float log2amp, __half* __restrict__ Ksh, int Npad, float* __restrict__ mun, int store_tiles /* trial tiles whose K* columns are written */) {
  extern __shared__ unsigned char ks_smem_raw[];
  unsigned char* base = (unsigned char*)(((uintptr_t)ks_smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* smA = base;                                            // [ns][hi 8 KB | lo 8 KB]
  unsigned char* ring = smA + (size_t)ns * 2 * KS_A_PLANE_BYTES;        // [KS_STAGES][hi 8 KB | lo 8 KB]
  unsigned char* nxs = ring + KS_STAGES * KS_STAGE_BYTES;               // [KS_STAGES][1 KB of pairs], entry t % KS_STAGES
  KsSmem* S = (KsSmem*)(nxs + KS_STAGES * KS_NX_BYTES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * KS_BM;

  if (threadIdx.x == KS_CONSUMERS) {
    prefetch_tmap(&tmCh);
    prefetch_tmap(&tmCl);
    prefetch_tmap(&tmXh);
    prefetch_tmap(&tmXl);
    for (int i = 0; i < KS_STAGES; i++) {
      mbar_init(smem_u32(&S->full[i]), 1);
      mbar_init(smem_u32(&S->empty[i]), 2);   // one arrive per consumer warpgroup
    }
    mbar_init(smem_u32(&S->a_full), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == KS_CONSUMERS / 32) {
    // ===================================== TMA producer ===========================================
    if (lane == 0) {
      const uint32_t abar = smem_u32(&S->a_full);
      mbar_expect_tx(abar, (uint32_t)ns * 2 * KS_A_PLANE_BYTES);
      for (int sl = 0; sl < ns; sl++) {
        tma_load_2d(smem_u32(smA + (size_t)sl * 2 * KS_A_PLANE_BYTES), &tmCh, abar, sl * KS_BK, m0);
        tma_load_2d(smem_u32(smA + (size_t)sl * 2 * KS_A_PLANE_BYTES + KS_A_PLANE_BYTES), &tmCl, abar, sl * KS_BK, m0);
      }
      uint32_t c = 0;
      for (int t = 0; t < ntiles; t++)
        for (int sl = 0; sl < ns; sl++, c++) {
          const uint32_t st = c % KS_STAGES, use = c / KS_STAGES;
          mbar_wait(smem_u32(&S->empty[st]), (use & 1) ^ 1);
          const uint32_t bar = smem_u32(&S->full[st]);
          const bool pairs = sl == 0 && t < nx_tiles;   // tiles past the trials' extent have no pairs: the EDGE body masks them
          mbar_expect_tx(bar, KS_STAGE_BYTES + (pairs ? KS_NX_BYTES : 0));
          const uint32_t dst = smem_u32(ring + (size_t)st * KS_STAGE_BYTES);
          tma_load_2d(dst, &tmXh, bar, sl * KS_BK, t * KS_BN);
          tma_load_2d(dst + KS_B_PLANE_BYTES, &tmXl, bar, sl * KS_BK, t * KS_BN);
          if (pairs) bulk_load(smem_u32(nxs + (size_t)(t % KS_STAGES) * KS_NX_BYTES), nxal4 + (size_t)t * (KS_BN / 2), KS_NX_BYTES, bar);
        }
    }
    __syncwarp();
  } else {
    // ===================================== consumer warpgroups ====================================
    // Both warpgroups run their MMAs and then their epilogues at the same time.  Alternating them (one warpgroup's MMAs under the
    // other's epilogue, by named turn barriers) was slower on an H100: tests/studies/kstar_probe.cu, and DESIGN.md §3.
    const int wg = threadIdx.x >> 7, wl = (threadIdx.x >> 5) & 3, q = lane & 3;
    const int r0 = m0 + wg * 64 + wl * 16 + (lane >> 2), r1 = r0 + 8;
    const bool signal = (threadIdx.x & 127) == 0;
    // Each tile's (|x̂|², alpha) pairs sit in ring entry t % KS_STAGES until the producer refills it for tile t + KS_STAGES.  With
    // one slab per tile that refill waits on this tile's own stage, so the stage is released only after the whole warpgroup has
    // read the pairs (warpgroup barrier 1 + wg).  With more slabs it waits on a slab of tile t + 2 or later, released after that
    // same barrier of tile t.
    const bool hold = ns == 1;
    const float nc0 = ncand[r0], nc1 = ncand[r1];
    __half* out0 = Ksh + (size_t)r0 * Npad;
    __half* out1 = Ksh + (size_t)r1 * Npad;
    double mu0 = 0.0, mu1 = 0.0;
    float acc[64];
    mbar_wait(smem_u32(&S->a_full), 0);
    uint32_t c = 0;
    for (int t = 0; t < ntiles; t++) {
      int pending = -1;
      for (int sl = 0; sl < ns; sl++, c++) {
        const uint32_t st = c % KS_STAGES, use = c / KS_STAGES;
        mbar_wait(smem_u32(&S->full[st]), use & 1);
        const uint32_t a_hi = smem_u32(smA + (size_t)sl * 2 * KS_A_PLANE_BYTES) + wg * (KS_A_PLANE_BYTES / 2), a_lo = a_hi + KS_A_PLANE_BYTES;
        const uint32_t b_hi = smem_u32(ring + (size_t)st * KS_STAGE_BYTES), b_lo = b_hi + KS_B_PLANE_BYTES;
        wgmma_fence();
        // small products first: the accumulator is still tiny when they are added, so their bits are not truncated away
#pragma unroll
        for (int prod = 0; prod < 4; prod++) {
          const uint32_t a = (prod < 2) ? a_lo : a_hi;
          const uint32_t b = (prod & 1) ? b_hi : b_lo;   // lo·lo, lo·hi, hi·lo, hi·hi
#pragma unroll
          for (int k = 0; k < KS_BK / 16; k++)
            wgmma_f16_n128(acc, gmma_desc_sw64(a + k * 32), gmma_desc_sw64(b + k * 32), (sl > 0 || prod > 0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (pending >= 0 && signal) mbar_arrive(smem_u32(&S->empty[pending]));
        pending = (int)st;
      }
      wgmma_wait<0>();
      acc_fence(acc);
      if (!hold && signal) mbar_arrive(smem_u32(&S->empty[pending]));   // the accumulator is in registers; the pairs have their own ring
      const uint32_t nx = smem_u32(nxs + (size_t)(t % KS_STAGES) * KS_NX_BYTES) + q * 16;
      const int n_base = t * KS_BN;
      // EDGE: only the last tile(s) mask trials >= N.  STORE: a pruning pass contracts a prefix of the trials only, so tiles past
      // store_tiles feed the mean and write no K* columns.  Instantiations behind warp-uniform branches keep the mask, and the
      // conversions, addresses and stores, out of the per-element code of the tiles that do not need them.
      auto tile_body = [&](auto edge_tag, auto store_tag) {
        constexpr bool EDGE = decltype(edge_tag)::value, STORE = decltype(store_tag)::value;
        float ma0 = 0.f, mb0 = 0.f, ma1 = 0.f, mb1 = 0.f;   // two fp32 chains per row, added in FP64 once per tile
#pragma unroll
        for (int i = 0; i < KS_BN / 8; i++) {
          const int n = n_base + 8 * i + 2 * q;
          const float4 na = (EDGE && n >= N) ? make_float4(0.f, 0.f, 0.f, 0.f) : lds128(nx + i * 64);
          float k00 = ks_kernel_value<KIND>(acc[4 * i], nc0 + na.x, log2amp);
          float k01 = ks_kernel_value<KIND>(acc[4 * i + 1], nc0 + na.z, log2amp);
          float k10 = ks_kernel_value<KIND>(acc[4 * i + 2], nc1 + na.x, log2amp);
          float k11 = ks_kernel_value<KIND>(acc[4 * i + 3], nc1 + na.z, log2amp);
          if (EDGE) {
            k00 = n < N ? k00 : 0.f;
            k10 = n < N ? k10 : 0.f;
            k01 = n + 1 < N ? k01 : 0.f;
            k11 = n + 1 < N ? k11 : 0.f;
          }
          ma0 = fmaf(k00, na.y, ma0);
          mb0 = fmaf(k01, na.w, mb0);
          ma1 = fmaf(k10, na.y, ma1);
          mb1 = fmaf(k11, na.w, mb1);
          if (STORE) {
            *reinterpret_cast<__half2*>(out0 + n) = __floats2half2_rn(k00, k01);
            *reinterpret_cast<__half2*>(out1 + n) = __floats2half2_rn(k10, k11);
          }
        }
        mu0 += (double)(ma0 + mb0);
        mu1 += (double)(ma1 + mb1);
      };
      const bool edge = n_base + KS_BN > N;
      if (t < store_tiles) {
        if (edge)
          tile_body(std::true_type{}, std::true_type{});
        else
          tile_body(std::false_type{}, std::true_type{});
      } else {
        if (edge)
          tile_body(std::true_type{}, std::false_type{});
        else
          tile_body(std::false_type{}, std::false_type{});
      }
      named_bar_sync(1 + wg, 128);   // every warp of this warpgroup is done with the tile's pairs
      if (hold && signal) mbar_arrive(smem_u32(&S->empty[pending]));
    }
    // the four lanes of a quad hold the same two rows: fixed-order butterfly
    mu0 += __shfl_xor_sync(0xffffffffu, mu0, 1);
    mu1 += __shfl_xor_sync(0xffffffffu, mu1, 1);
    mu0 += __shfl_xor_sync(0xffffffffu, mu0, 2);
    mu1 += __shfl_xor_sync(0xffffffffu, mu1, 2);
    if (q == 0) {
      mun[r0] = (float)mu0;
      mun[r1] = (float)mu1;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Operand preparation.  x̂ = (x/ℓ − centre)·kscale, clamped to ±32768 (fp16 range; anything that far from the trials has
// k = 0 either way), hi = fp16(x̂), lo = fp16(x̂ − hi); the squared norm is taken of hi + lo, the point the MMAs actually see.
__global__ void __launch_bounds__(256) ks_center_kernel(const double* __restrict__ XsT, int ldx, int N, double* __restrict__ center) {
  __shared__ double red[256];
  const double* col = XsT + (size_t)blockIdx.x * ldx;
  double a = 0.0;
  for (int i = threadIdx.x; i < N; i += 256) a += col[i];
  red[threadIdx.x] = a;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) center[blockIdx.x] = red[0] / N;
}

__device__ __forceinline__ void ks_split(double v, __half& hi, __half& lo, double& seen) {
  v = fmin(fmax(v, -32768.0), 32768.0);
  hi = __double2half(v);
  lo = __double2half(v - (double)__half2float(hi));
  seen = (double)__half2float(hi) + (double)__half2float(lo);
}

// one warp per row; rows >= n_valid and features >= D are written as zeros (planes are rows_pad × Dp)
template <typename XT, bool SCALED /* input already divided by ℓ (the trials' Xs) */>
__global__ void __launch_bounds__(256)
ks_split_rows_kernel(const XT* __restrict__ X, int64_t n_valid, int64_t rows_pad, int D, int Dp, const double* __restrict__ inv_ls, int n_ls,
                     const double* __restrict__ center, double kscale, __half* __restrict__ Ph, __half* __restrict__ Pl, float* __restrict__ nrm,
                     int nrm_stride, const double* __restrict__ alpha /* trials: second float of the (norm, alpha) pair */) {
  const int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows_pad) return;
  double s = 0.0;
  for (int d = lane; d < Dp; d += 32) {
    __half hi = __float2half(0.f), lo = hi;
    if (r < n_valid && d < D) {
      double v = (double)X[r * D + d];
      if (!SCALED) v *= inv_ls[n_ls == 1 ? 0 : d];
      double seen;
      ks_split((v - center[d]) * kscale, hi, lo, seen);
      s = fma(seen, seen, s);
    }
    Ph[r * Dp + d] = hi;
    Pl[r * Dp + d] = lo;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    nrm[r * nrm_stride] = (float)s;
    if (alpha) nrm[r * nrm_stride + 1] = r < n_valid ? (float)alpha[r] : 0.f;
  }
}

}  // namespace

static double ks_kscale(int kind) { return kind == KBO_KERNEL_RBF ? 0.70710678118654752440 : 2.23606797749978969641; }

// Trial-side operands of the tensor-core K* kernel: planes of the centred, scaled trials and the (|x̂|², alpha) pairs.  Cheap
// (N·D); redone by every fit / append / rebase finish because alpha changes with each of them.
int kbo_i_tc_trials_prep(kbo_handle* h, bool new_center, cudaStream_t s) {
  const int N = h->N, D = h->D, Dp = round_up(D, KS_BK), Np = round_up(N, KS_BN);
  h->ks_ready = false;
  if (D > KS_MAX_SLABS * KS_BK) return KBO_OK;   // the FP64 K* kernel serves wider spaces
  KBO_TRY(kbo_reserve(h, h->ks_center, 512));
  KBO_TRY(kbo_reserve(h, h->ks_Xh, (size_t)Np * Dp));
  KBO_TRY(kbo_reserve(h, h->ks_Xl, (size_t)Np * Dp));
  KBO_TRY(kbo_reserve(h, h->ks_nxal, (size_t)Np * 2));
  if (new_center) {
    ks_center_kernel<<<D, 256, 0, s>>>(h->XsT.p, h->ld, N, h->ks_center.p);
    KBO_LAUNCH_CHECK(h);
  }
  ks_split_rows_kernel<double, true><<<(unsigned)((Np + 7) / 8), 256, 0, s>>>(h->Xs.p, N, Np, D, Dp, nullptr, 1, h->ks_center.p,
                                                                          ks_kscale(h->prm.kernel), h->ks_Xh.p, h->ks_Xl.p,
                                                                          h->ks_nxal.p, 2, h->alpha.p);
  KBO_LAUNCH_CHECK(h);
  h->ks_ready = true;
  return KBO_OK;
}

// K̃* hi plane (rows_pad × Npad fp16, rows_pad = rows rounded up to 256) and μ̃ for `rows` candidates starting at Xc.
int kbo_i_tc_kstar(kbo_handle* h, const void* Xc, int xc_dtype, int64_t rows, __half* Ksh, float* mun, cudaStream_t s, int store_cols) {
  if (!h->ks_ready) KBO_FAIL(h, KBO_ERR_STATE, "tc_kstar: trial operands not prepared");
  const int N = h->N, D = h->D, Dp = round_up(D, KS_BK), Np = round_up(N, KS_BN), ns = Dp / KS_BK;
  const int64_t rows_pad = round_up64(rows, 256);
  if (h->Npad % KS_BN != 0 || h->Npad < Np) KBO_FAIL(h, KBO_ERR_STATE, "tc_kstar: Npad %d does not cover N %d", h->Npad, N);
  KBO_TRY(kbo_reserve(h, h->ks_Ch, (size_t)rows_pad * Dp));
  KBO_TRY(kbo_reserve(h, h->ks_Cl, (size_t)rows_pad * Dp));
  KBO_TRY(kbo_reserve(h, h->ks_nc, (size_t)rows_pad));
  const unsigned g = (unsigned)((rows_pad + 7) / 8);
  if (xc_dtype == KBO_F64)
    ks_split_rows_kernel<double, false><<<g, 256, 0, s>>>((const double*)Xc, rows, rows_pad, D, Dp, h->d_inv_ls.p, (int)h->inv_ls.size(),
                                                         h->ks_center.p, ks_kscale(h->prm.kernel), h->ks_Ch.p, h->ks_Cl.p,
                                                         h->ks_nc.p, 1, nullptr);
  else
    ks_split_rows_kernel<float, false><<<g, 256, 0, s>>>((const float*)Xc, rows, rows_pad, D, Dp, h->d_inv_ls.p, (int)h->inv_ls.size(),
                                                        h->ks_center.p, ks_kscale(h->prm.kernel), h->ks_Ch.p, h->ks_Cl.p,
                                                        h->ks_nc.p, 1, nullptr);
  KBO_LAUNCH_CHECK(h);
  CUtensorMap tmCh, tmCl, tmXh, tmXl;
  KBO_TRY(kbo_i_encode_map_f16(h, &tmCh, h->ks_Ch.p, (uint64_t)Dp, (uint64_t)rows_pad, KS_BK, KS_BM));
  KBO_TRY(kbo_i_encode_map_f16(h, &tmCl, h->ks_Cl.p, (uint64_t)Dp, (uint64_t)rows_pad, KS_BK, KS_BM));
  KBO_TRY(kbo_i_encode_map_f16(h, &tmXh, h->ks_Xh.p, (uint64_t)Dp, (uint64_t)Np, KS_BK, KS_BN));
  KBO_TRY(kbo_i_encode_map_f16(h, &tmXl, h->ks_Xl.p, (uint64_t)Dp, (uint64_t)Np, KS_BK, KS_BN));
  const size_t smem = ks_smem_bytes(ns);
  const float log2amp = (float)log2(h->prm.amplitude);
  const int ntiles = h->Npad / KS_BN;   // tiles past Np read out-of-bounds trial rows (TMA zero fill) and are masked to 0
  const int store_tiles = (store_cols < 0 || store_cols >= h->Npad) ? ntiles : (store_cols + KS_BN - 1) / KS_BN;
  // two trials' (|x̂|², alpha) pairs per float4: device allocations are 256-byte aligned, so each group of four floats is 16-byte aligned
  const float4* nxal = reinterpret_cast<const float4*>(h->ks_nxal.p);
  if (h->prm.kernel == KBO_KERNEL_RBF) {
    KBO_CUDA(h, cudaFuncSetAttribute(tc_kstar_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    tc_kstar_kernel<0><<<(unsigned)(rows_pad / KS_BM), KS_THREADS, smem, s>>>(tmCh, tmCl, tmXh, tmXl, ns, ntiles, N, h->ks_nc.p,
                                                                            nxal, Np / KS_BN, log2amp, Ksh, h->Npad, mun, store_tiles);
  } else {
    KBO_CUDA(h, cudaFuncSetAttribute(tc_kstar_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    tc_kstar_kernel<1><<<(unsigned)(rows_pad / KS_BM), KS_THREADS, smem, s>>>(tmCh, tmCl, tmXh, tmXl, ns, ntiles, N, h->ks_nc.p,
                                                                            nxal, Np / KS_BN, log2amp, Ksh, h->Npad, mun, store_tiles);
  }
  KBO_LAUNCH_CHECK(h);
  return KBO_OK;
}
