// Ranking pass of the variance contraction on the Hopper tensor cores (sm_90a: wgmma + TMA + mbarrier).
//
//   Σ_j ṽ[m,j]²,   ṽ[m,j] = Σ_{k≤j} K̃*h[m,k]·Wh[j,k]          (hi planes only: ONE fp16 product per term, $SK/_gpr.py:460,:480)
//
// Work item = (128-row group, pair of 256-column j-tiles); the K range of tile t is its triangular extent k < 256·(t+1).  Items
// are dealt to persistent CTAs (one per SM) in row-group-major order, so the CTAs running at any moment work on neighbouring
// row groups: their K* rows and the part of W's triangle in use stay in the 50 MB L2 and each K* byte is read from DRAM about
// once.  No intermediate drains: a ranking pass does not care about the truncation of long fp32 accumulation chains, so each
// accumulator is read once per tile.
//   warps 0-7  two consumer warpgroups: rows 64·wg … 64·wg + 63 of the item, wgmma m64n256k16 into 128 fp32 registers per
//              thread, then Σ v² per row → part[pair][row]
//   warp 8     TMA producer (one thread): A (K̃*, 128 × 32) and B (W, 256 × 32) per stage, SWIZZLE_64B, 8-stage ring
#include "kbo_internal.cuh"
#include "tc_common.cuh"

#define RK_BM 128
#define RK_BN 256
#define RK_BK 32
#define RK_STAGES 8
#define RK_A_BYTES (RK_BM * RK_BK * 2)           // 8 KB
#define RK_B_BYTES (RK_BN * RK_BK * 2)           // 16 KB
#define RK_STAGE_BYTES (RK_A_BYTES + RK_B_BYTES)
#define RK_CONSUMERS 256                         // two warpgroups
#define RK_THREADS (RK_CONSUMERS + 32)
#define RK_SMEM_BYTES (1024 + RK_STAGES * RK_STAGE_BYTES + 256)
#define RK_CPT (RK_BN / RK_BK)                   // chunks per 256 trials

namespace {
using namespace tcx;

struct RkSmem {
  uint64_t full[RK_STAGES];
  uint64_t empty[RK_STAGES];
};

struct RkItem {
  int rg, p, t0, ntiles;
};
// Work item (128-row group rg, tile pair p).  The item lists are built on the host (rk_schedule below): every role of a CTA
// walks the same list sched[off[c] .. off[c+1]).
__device__ __forceinline__ RkItem rk_item(int code, int n_jtiles) {
  RkItem w;
  w.rg = code >> 8;
  w.p = code & 255;
  w.t0 = 2 * w.p;
  w.ntiles = w.t0 + 1 < n_jtiles ? 2 : 1;
  return w;
}

__global__ void __launch_bounds__(RK_THREADS, 1)
tc_rank_kernel(const __grid_constant__ CUtensorMap tmA /* K̃* hi plane, box 32 × 128 */, const __grid_constant__ CUtensorMap tmW /* W hi plane, box 32 × 256 */,
               int n_jtiles, const int* __restrict__ sched /* [n_ctas + 1 offsets | item codes] */, float* __restrict__ part /* [n_pairs][rows] Σ v² over the pair's 512 columns (scaled units) */,
               int64_t rows) {
  extern __shared__ unsigned char rk_smem_raw[];
  unsigned char* ring = (unsigned char*)(((uintptr_t)rk_smem_raw + 1023) & ~(uintptr_t)1023);
  RkSmem* S = (RkSmem*)(ring + RK_STAGES * RK_STAGE_BYTES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int it_begin = __ldg(sched + blockIdx.x), it_end = __ldg(sched + blockIdx.x + 1);

  if (threadIdx.x == RK_CONSUMERS) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmW);
    for (int i = 0; i < RK_STAGES; i++) {
      mbar_init(smem_u32(&S->full[i]), 1);    // the producer's expect_tx; the bytes complete the phase
      mbar_init(smem_u32(&S->empty[i]), 2);   // one arrive per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == RK_CONSUMERS / 32) {
    // ===================================== TMA producer ==========================================
    if (lane == 0) {
      uint32_t c = 0;
      for (int it = it_begin; it < it_end; it++) {
        const RkItem w = rk_item(__ldg(sched + it), n_jtiles);
        const int m0 = w.rg * RK_BM;
        for (int tt = 0; tt < w.ntiles; tt++) {
          const int t = w.t0 + tt, nch = (t + 1) * RK_CPT;
          for (int ch = 0; ch < nch; ch++, c++) {
            const uint32_t st = c % RK_STAGES, use = c / RK_STAGES;
            mbar_wait(smem_u32(&S->empty[st]), (use & 1) ^ 1);
            const uint32_t bar = smem_u32(&S->full[st]);
            mbar_expect_tx(bar, RK_STAGE_BYTES);
            const uint32_t dst = smem_u32(ring + (size_t)st * RK_STAGE_BYTES);
            tma_load_2d(dst, &tmA, bar, ch * RK_BK, m0);
            tma_load_2d(dst + RK_A_BYTES, &tmW, bar, ch * RK_BK, t * RK_BN);
          }
        }
      }
    }
    __syncwarp();
  } else {
    // ===================================== consumer warpgroups ===================================
    const int wg = threadIdx.x >> 7, wl = (threadIdx.x >> 5) & 3;
    const int row0 = wg * 64 + wl * 16 + (lane >> 2);   // and row0 + 8
    const bool signal = (threadIdx.x & 127) == 0;
    float acc[128];
    uint32_t c = 0;
    for (int it = it_begin; it < it_end; it++) {
      const RkItem w = rk_item(__ldg(sched + it), n_jtiles);
      float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;   // rows row0 (s0, s1) and row0 + 8 (s2, s3)
      for (int tt = 0; tt < w.ntiles; tt++) {
        const int nch = (w.t0 + tt + 1) * RK_CPT;
        uint32_t prev = 0;
        for (int ch = 0; ch < nch; ch++, c++) {
          const uint32_t st = c % RK_STAGES, use = c / RK_STAGES;
          mbar_wait(smem_u32(&S->full[st]), use & 1);
          const uint32_t a = smem_u32(ring + (size_t)st * RK_STAGE_BYTES) + wg * (RK_A_BYTES / 2), b = smem_u32(ring + (size_t)st * RK_STAGE_BYTES) + RK_A_BYTES;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < RK_BK / 16; k++) wgmma_f16_n256(acc, gmma_desc_sw64(a + k * 32), gmma_desc_sw64(b + k * 32), (ch > 0 || k > 0) ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();   // the previous chunk's MMAs are done: its stage may be refilled
          if (ch > 0 && signal) mbar_arrive(smem_u32(&S->empty[prev]));
          prev = st;
        }
        wgmma_wait<0>();
        acc_fence(acc);
        if (signal) mbar_arrive(smem_u32(&S->empty[prev]));
#pragma unroll
        for (int i = 0; i < 128; i += 4) {
          s0 = fmaf(acc[i], acc[i], s0);
          s1 = fmaf(acc[i + 1], acc[i + 1], s1);
          s2 = fmaf(acc[i + 2], acc[i + 2], s2);
          s3 = fmaf(acc[i + 3], acc[i + 3], s3);
        }
      }
      float r0 = s0 + s1, r1 = s2 + s3;   // the four lanes of a quad hold the same two rows: fixed-order butterfly
      r0 += __shfl_xor_sync(0xffffffffu, r0, 1);
      r1 += __shfl_xor_sync(0xffffffffu, r1, 1);
      r0 += __shfl_xor_sync(0xffffffffu, r0, 2);
      r1 += __shfl_xor_sync(0xffffffffu, r1, 2);
      if ((lane & 3) == 0) {
        float* out = part + (size_t)w.p * rows + (size_t)w.rg * RK_BM;
        out[row0] = r0;
        out[row0 + 8] = r1;
      }
    }
  }
}

__global__ void rank_finish_kernel(const float* __restrict__ part, int p_begin, int p_end, int64_t rows, const double* __restrict__ w_scale, double amp,
                                   float* __restrict__ var_out) {
  const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= rows) return;
  double tot = 0.0;
  for (int p = p_begin; p < p_end; p++) tot += (double)part[(size_t)p * rows + m];
  const double sc = w_scale[1];
  var_out[m] = (float)(amp - tot * sc * sc);
}

// Item lists: items in row-group-major order (largest tile pair of a group first), each dealt to the least-loaded CTA.  Loads
// stay level, and because they do, the CTAs consume the row groups in step: the items in flight always belong to a few
// neighbouring row groups, whose K* rows therefore stay in L2.
int rk_schedule(kbo_handle* h, int n_rg, int n_jtiles, int ctas, int p_begin, int p_end, const int** sched_dev, cudaStream_t s) {
  for (auto& e : h->rk_sched)
    if (e.key[0] == n_rg && e.key[1] == n_jtiles && e.key[2] == ctas && e.key[3] == p_begin && e.key[4] == p_end) {
      *sched_dev = e.dev.p;
      return KBO_OK;
    }
  kbo_handle::RkSched& e = h->rk_sched[h->rk_sched_next];
  h->rk_sched_next = (h->rk_sched_next + 1) % 8;
  e.key[0] = -1;
  std::vector<std::vector<int>> lists(ctas);
  std::vector<long long> load(ctas, 0);
  for (int rg = 0; rg < n_rg; rg++)
    for (int p = p_end - 1; p >= p_begin; p--) {
      int best = 0;
      for (int c = 1; c < ctas; c++)
        if (load[c] < load[best]) best = c;
      const bool live1 = 2 * p + 1 < n_jtiles;
      load[best] += (2 * p + 1) * RK_CPT + (live1 ? (2 * p + 2) * RK_CPT : 0) + 3;   // MMA chunk-units + the drain
      lists[best].push_back((rg << 8) | p);
    }
  e.host.assign(ctas + 1, 0);
  int off = ctas + 1;
  for (int c = 0; c < ctas; c++) {
    e.host[c] = off;
    off += (int)lists[c].size();
  }
  e.host[ctas] = off;
  for (int c = 0; c < ctas; c++) e.host.insert(e.host.end(), lists[c].begin(), lists[c].end());
  KBO_TRY(kbo_reserve(h, e.dev, e.host.size()));
  // pageable source: the runtime stages it before returning, and earlier launches reading this buffer precede the copy on s
  KBO_CUDA(h, kbo_copy(e.dev.p, e.host.data(), e.host.size(), cudaMemcpyHostToDevice, s));
  e.key[0] = n_rg;
  e.key[1] = n_jtiles;
  e.key[2] = ctas;
  e.key[3] = p_begin;
  e.key[4] = p_end;
  *sched_dev = e.dev.p;
  return KBO_OK;
}

}  // namespace

// var_n_out[m] = amp − Σ_j (Σ_k K̃*h[m,k]·W[j,k])² for `rows` (multiple of 256) candidate rows of the hi plane Ksh (rows × Npad),
// j restricted to the tile pairs [p_begin, p_end) (p_end < 0: all).  A PREFIX of the pairs gives an upper bound on the variance
// (every (W k*)_j² is non-negative) at the cost of the prefix's share of the triangle: the first eighth of the trials costs 1/64.
int kbo_i_tc_rank(kbo_handle* h, const __half* Ksh, int64_t rows, const __half* Wh, int Npad, double amp, float* var_n_out, cudaStream_t s,
                  int p_begin, int p_end) {
  if (rows % 256 != 0 || Npad % RK_BN != 0) KBO_FAIL(h, KBO_ERR_INVALID, "tc_rank: rows %% 256 and Npad %% 256 must be 0");
  CUtensorMap tmA, tmW;
  KBO_TRY(kbo_i_encode_map_f16(h, &tmA, Ksh, (uint64_t)Npad, (uint64_t)rows, RK_BK, RK_BM));
  KBO_TRY(kbo_i_encode_map_f16(h, &tmW, Wh, (uint64_t)Npad, (uint64_t)Npad, RK_BK, RK_BN));
  if (!h->attr_rank) {
    KBO_CUDA(h, cudaFuncSetAttribute(tc_rank_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, RK_SMEM_BYTES));
    h->attr_rank = true;
  }
  const int n_jtiles = Npad / RK_BN, n_pairs = (n_jtiles + 1) / 2;
  const int64_t n_rg = rows / RK_BM;
  if (p_end < 0 || p_end > n_pairs) p_end = n_pairs;
  if (p_begin < 0 || p_begin >= p_end) KBO_FAIL(h, KBO_ERR_INVALID, "tc_rank: empty tile-pair range [%d, %d)", p_begin, p_end);
  if (n_pairs > 256 || n_rg >= (1 << 23)) KBO_FAIL(h, KBO_ERR_INVALID, "tc_rank: problem too large for the item encoding (Npad %d, rows %lld)", Npad, (long long)rows);
  KBO_TRY(kbo_reserve(h, h->rk_part, (size_t)n_pairs * rows));
  int ctas = h->sm_count;
  if ((int64_t)ctas > n_rg * (p_end - p_begin)) ctas = (int)(n_rg * (p_end - p_begin));
  const int* sched = nullptr;
  KBO_TRY(rk_schedule(h, (int)n_rg, n_jtiles, ctas, p_begin, p_end, &sched, s));
  tc_rank_kernel<<<(unsigned)ctas, RK_THREADS, RK_SMEM_BYTES, s>>>(tmA, tmW, n_jtiles, sched, h->rk_part.p, rows);
  KBO_LAUNCH_CHECK(h);
  rank_finish_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, s>>>(h->rk_part.p, p_begin, p_end, rows, h->scal.p + S_WSCALE, amp, var_n_out);
  KBO_LAUNCH_CHECK(h);
  return KBO_OK;
}
