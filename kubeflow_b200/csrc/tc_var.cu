// Variance contraction on the Hopper tensor cores (wgmma + TMA + mbarrier, 2-CTA clusters), sm_90a.
//
//   var_n[m] = amp − Σ_j v[m,j]²,   v[m,j] = Σ_{k≤j} K*[m,k]·W[j,k]      ($SK/_gpr.py:460, :480-481 with W = L⁻¹)
//
// This is the M·N² term that sets the suggestion rate (SURVEY.md §8(d)).  Operands are fp16 hi/lo splits
// (x ≈ hi + lo, |x − hi − lo| ≤ 2⁻²²|x|) and each product is three MMAs  Ah·Bh + Ah·Bl + Al·Bh  into one
// fp32 accumulator: bf16/fp16 single-pass moves σ² by 1e-2 and bf16×3 by 1e-5..1e-4 (DESIGN.md §numerics) — fp16×3
// stays at ~3e-7.
//
// A 2-CTA cluster per 128-row panel, j-tiles split by parity, K* chunks TMA-multicast to both CTAs.
// CTA = 128 candidate rows × its j-tiles of 128 trial columns, walked in order; for j-tile t only k < 128(t+1) is issued (W is
// lower triangular).  K is consumed in 32-wide chunks through a 6-stage TMA→smem ring:
//   warps 0-7  two consumer warpgroups (rows 64·wg …): wgmma m64n128k16 into 64 fp32 registers per thread.  Every `k_span`
//              trials the accumulator is added into a second register array with round-to-nearest — this bounds the length
//              of the tensor-core accumulation chain — and Σv² per row is taken at the end of each j-tile.
//   warp 8     TMA producer (A hi/lo 128×32, B hi/lo 128×32 per stage, SWIZZLE_64B, mbarrier expect_tx)
#include <cuda.h>
#include <stdlib.h>

#include "kbo_internal.cuh"
#include "tc_common.cuh"

#define TC_BM 128
#define TC_BN 128
#define TC_BK 32
#define TC_CPT (TC_BN / TC_BK)                // chunks per j-tile of K
#define TC_STAGES 6
#define TC_A_BYTES (TC_BM * TC_BK * 2)        // 8 KB per plane
#define TC_B_BYTES (TC_BN * TC_BK * 2)        // 8 KB per plane
#define TC_STAGE_BYTES (2 * TC_A_BYTES + 2 * TC_B_BYTES)  // 32 KB
#define TC_CONSUMERS 256
#define TC_THREADS (TC_CONSUMERS + 32)
#define TC_SMEM_BYTES (TC_STAGES * TC_STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/)

namespace {
using namespace tcx;

struct TcSmem {
  uint64_t full[TC_STAGES];
  uint64_t empty[TC_STAGES];
};

// The j-tiles are split by parity (CTA r owns tiles 2p + r) and both CTAs walk the K chunks of a tile pair in lockstep, so
// every A (K*) chunk is fetched ONCE and TMA-multicast into both CTAs' shared memory (each CTA issues the load for its 64-row
// half with ctaMask = 0b11); B (W) chunks stay private.  That halves the K* panel re-reads.
//   full[st]  (per CTA): 1 arrival (own producer's expect_tx) + A bytes from both multicast halves + own B bytes
//   empty[st] (per CTA): one arrival per consumer warpgroup of BOTH CTAs, so a stage is refilled only when both CTAs are done
// Per-row Σv² of the two CTAs' tile sets goes to part[rank][row]; tc_variance_finish_kernel adds them in a fixed order.
// nprod 3: Al·Bh + Ah·Bl + Ah·Bh; 1: Ah·Bh only (ranking pass, lo planes never loaded).
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_variance_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
                   const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl, int n_jtiles,
                   int span_chunks, int nprod, double* __restrict__ part /* [2][rows] raw Σv² (scaled units) */, int64_t rows) {
  extern __shared__ unsigned char tc_smem_raw[];
  // SWIZZLE_64B tiles need 512 B alignment of each plane; keep the whole ring 1024 B aligned.
  unsigned char* ring = (unsigned char*)(((uintptr_t)tc_smem_raw + 1023) & ~(uintptr_t)1023);
  TcSmem* S = (TcSmem*)(ring + TC_STAGES * TC_STAGE_BYTES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = cluster_ctarank();
  const int m0 = (blockIdx.x >> 1) * TC_BM;
  const int n_groups = (n_jtiles + 1) / 2;
  const uint32_t planes = nprod == 3 ? 2u : 1u;

  if (threadIdx.x == TC_CONSUMERS) {
    prefetch_tmap(&tmAh);
    prefetch_tmap(&tmAl);
    prefetch_tmap(&tmBh);
    prefetch_tmap(&tmBl);
    for (int i = 0; i < TC_STAGES; i++) {
      mbar_init(smem_u32(&S->full[i]), 1);
      mbar_init(smem_u32(&S->empty[i]), 4);   // two consumer warpgroups in each of the two CTAs
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  cluster_sync_all();  // the peer's barriers exist before anything is multicast into them

  if (warp == TC_CONSUMERS / 32) {
    // ===================================== TMA producer ===========================================
    if (lane == 0) {
      uint32_t c = 0;
      for (int p = 0; p < n_groups; p++) {
        const int my_tile = 2 * p + (int)rank;
        const int my_nch = my_tile < n_jtiles ? (my_tile + 1) * TC_CPT : 0;
        const int nch = min(2 * p + 2, n_jtiles) * TC_CPT;  // a pair streams the longer of its two K ranges
        for (int ch = 0; ch < nch; ch++, c++) {
          const uint32_t st = c % TC_STAGES, use = c / TC_STAGES;
          mbar_wait_cluster(smem_u32(&S->empty[st]), (use & 1) ^ 1);
          const uint32_t bar = smem_u32(&S->full[st]);
          mbar_expect_tx(bar, planes * TC_A_BYTES + (ch < my_nch ? planes * TC_B_BYTES : 0));
          const uint32_t base = smem_u32(ring + st * TC_STAGE_BYTES);
          const int k0 = ch * TC_BK;
          const uint32_t half_off = rank * (TC_A_BYTES / 2);  // rows 64·rank … of the 128-row A tile
          tma_load_2d_mc(base + half_off, &tmAh, bar, k0, m0 + 64 * (int)rank, (uint16_t)3);
          if (nprod == 3) tma_load_2d_mc(base + TC_A_BYTES + half_off, &tmAl, bar, k0, m0 + 64 * (int)rank, (uint16_t)3);
          if (ch < my_nch) {
            tma_load_2d(base + 2 * TC_A_BYTES, &tmBh, bar, k0, my_tile * TC_BN);
            if (nprod == 3) tma_load_2d(base + 2 * TC_A_BYTES + TC_B_BYTES, &tmBl, bar, k0, my_tile * TC_BN);
          }
        }
      }
    }
    __syncwarp();
  } else {
    // ===================================== consumer warpgroups ====================================
    const int wg = threadIdx.x >> 7, wl = (threadIdx.x >> 5) & 3;
    const int row0 = wg * 64 + wl * 16 + (lane >> 2);  // and row0 + 8
    const bool signal = (threadIdx.x & 127) == 0;
    auto release = [&](uint32_t st) {
      if (!signal) return;
      mbar_arrive(smem_u32(&S->empty[st]));
      mbar_arrive_remote(smem_u32(&S->empty[st]), rank ^ 1u);
    };
    float acc[64], sum[64];
#pragma unroll
    for (int i = 0; i < 64; i++) sum[i] = 0.f;
    double rowacc0 = 0.0, rowacc1 = 0.0;
    uint32_t c = 0;
    for (int p = 0; p < n_groups; p++) {
      const int my_tile = 2 * p + (int)rank;
      const int my_nch = my_tile < n_jtiles ? (my_tile + 1) * TC_CPT : 0;
      const int nch = min(2 * p + 2, n_jtiles) * TC_CPT;
      for (int ch0 = 0; ch0 < nch; ch0 += span_chunks) {
        const int che = min(nch, ch0 + span_chunks);
        int pending = -1;   // stage whose MMAs are committed but not yet known complete
        for (int ch = ch0; ch < che; ch++, c++) {
          const uint32_t st = c % TC_STAGES, use = c / TC_STAGES;
          mbar_wait(smem_u32(&S->full[st]), use & 1);
          if (ch < my_nch) {
            const uint32_t base = smem_u32(ring + st * TC_STAGE_BYTES);
            const uint32_t ah = base + wg * (TC_A_BYTES / 2), al = ah + TC_A_BYTES;
            const uint32_t bh = base + 2 * TC_A_BYTES, bl = bh + TC_B_BYTES;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < TC_BK / 16; k++) {
              const uint32_t koff = k * 32;  // 16 fp16 = 32 B inside the 64 B swizzle row
              const uint32_t first = (ch > ch0 || k > 0) ? 1u : 0u;
              if (nprod == 3) {
                wgmma_f16_n128(acc, gmma_desc_sw64(al + koff), gmma_desc_sw64(bh + koff), first);  // small terms first
                wgmma_f16_n128(acc, gmma_desc_sw64(ah + koff), gmma_desc_sw64(bl + koff), 1u);
                wgmma_f16_n128(acc, gmma_desc_sw64(ah + koff), gmma_desc_sw64(bh + koff), 1u);
              } else {
                wgmma_f16_n128(acc, gmma_desc_sw64(ah + koff), gmma_desc_sw64(bh + koff), first);
              }
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (pending >= 0) release((uint32_t)pending);
            pending = (int)st;
          } else {   // the peer's tile needs this chunk, this CTA's does not
            wgmma_wait<0>();
            if (pending >= 0) release((uint32_t)pending);
            pending = -1;
            release(st);
          }
        }
        if (ch0 < my_nch) {   // this span holds MMAs of my tile: drain the accumulator
          wgmma_wait<0>();
          acc_fence(acc);
          if (pending >= 0) release((uint32_t)pending);
#pragma unroll
          for (int i = 0; i < 64; i++) sum[i] += acc[i];
        }
      }
      if (my_nch > 0) {
        // j-tile complete: Σ v² over this thread's 32 columns of each of its two rows (partial chains, then fp64 across tiles)
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
        for (int i = 0; i < 64; i += 4) {
          s0 = fmaf(sum[i], sum[i], s0);
          s1 = fmaf(sum[i + 1], sum[i + 1], s1);
          s2 = fmaf(sum[i + 2], sum[i + 2], s2);
          s3 = fmaf(sum[i + 3], sum[i + 3], s3);
          sum[i] = sum[i + 1] = sum[i + 2] = sum[i + 3] = 0.f;
        }
        rowacc0 += (double)(s0 + s1);
        rowacc1 += (double)(s2 + s3);
      }
    }
    // the four lanes of a quad hold the same two rows: fixed-order butterfly
    rowacc0 += __shfl_xor_sync(0xffffffffu, rowacc0, 1);
    rowacc1 += __shfl_xor_sync(0xffffffffu, rowacc1, 1);
    rowacc0 += __shfl_xor_sync(0xffffffffu, rowacc0, 2);
    rowacc1 += __shfl_xor_sync(0xffffffffu, rowacc1, 2);
    if ((lane & 3) == 0) {
      part[(size_t)rank * rows + m0 + row0] = rowacc0;
      part[(size_t)rank * rows + m0 + row0 + 8] = rowacc1;
    }
  }

  cluster_sync_all();  // no CTA leaves while its peer may still multicast into it or arrive on its barriers
}

__global__ void tc_variance_finish_kernel(const double* __restrict__ part, int64_t rows, const double* __restrict__ w_scale, double amp,
                                      float* __restrict__ var_out, double* __restrict__ sumsq_out) {
  const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= rows) return;
  const double sc = w_scale[1];
  const double tot = (part[m] + part[rows + m]) * sc * sc;
  var_out[m] = (float)(amp - tot);
  if (sumsq_out) sumsq_out[m] = tot;
}

int encode_map(kbo_handle* h, CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint32_t box_outer) {
  return kbo_i_encode_map_f16(h, out, base, inner, outer, TC_BK, box_outer);
}

int tc_launch(kbo_handle* h, const __half* Ksh, const __half* Ksl, int64_t rows, const __half* Wh, const __half* Wl, int Npad,
              const double* w_scale_dev, double amp, float* var_out, double* sumsq_out, int k_span, cudaStream_t s, int nprod = 3, int jtiles = -1) {
  // a prefix of the trial tiles (`jtiles` counts 256-column tiles): an upper bound on the variance
  const int n_jt = (jtiles > 0 && 2 * jtiles < Npad / TC_BN) ? 2 * jtiles : Npad / TC_BN;
  if (rows % TC_BM != 0 || Npad % 256 != 0) KBO_FAIL(h, KBO_ERR_INVALID, "tc_variance: rows %% 128 and Npad %% 256 must be 0");
  // Long tensor-core accumulation chains lose low-order bits; adding the accumulator into fp32 registers every 128 trials keeps
  // that error below the fp16×3 split error (≈ 5e-7).
  if (k_span <= 0) k_span = 128;
  int span_chunks = k_span / TC_BK;
  if (span_chunks < 1) span_chunks = 1;
  CUtensorMap tmAh, tmAl, tmBh, tmBl;
  // each CTA of a cluster loads (and multicasts) one 64-row half of the A tile
  KBO_TRY(encode_map(h, &tmAh, Ksh, (uint64_t)Npad, (uint64_t)rows, TC_BM / 2));
  KBO_TRY(encode_map(h, &tmAl, Ksl ? Ksl : Ksh, (uint64_t)Npad, (uint64_t)rows, TC_BM / 2));
  KBO_TRY(encode_map(h, &tmBh, Wh, (uint64_t)Npad, (uint64_t)Npad, TC_BN));
  KBO_TRY(encode_map(h, &tmBl, Wl ? Wl : Wh, (uint64_t)Npad, (uint64_t)Npad, TC_BN));
  if (!h->attr_tc) {
    KBO_CUDA(h, cudaFuncSetAttribute(tc_variance_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_BYTES));
    h->attr_tc = true;
  }
  // a 2-CTA cluster per 128-row panel: each K* chunk is read once for both CTAs (half the K* panel re-reads)
  KBO_TRY(kbo_reserve(h, h->part, (size_t)rows * 2));
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.gridDim = dim3((unsigned)(2 * (rows / TC_BM)));
  cfg.blockDim = dim3(TC_THREADS);
  cfg.dynamicSmemBytes = TC_SMEM_BYTES;
  cfg.stream = s;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  KBO_CUDA(h, cudaLaunchKernelEx(&cfg, tc_variance_kernel, tmAh, tmAl, tmBh, tmBl, n_jt, span_chunks, nprod, h->part.p, rows));
  KBO_LAUNCH_CHECK(h);
  tc_variance_finish_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, s>>>(h->part.p, rows, w_scale_dev, amp, var_out, sumsq_out);
  KBO_LAUNCH_CHECK(h);
  return KBO_OK;
}

}  // namespace

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// 2-D fp16 tensor map, row pitch = inner elements, box = box_inner × box_outer, SWIZZLE_64B (box_inner must be 32)
int kbo_i_encode_map_f16(kbo_handle* h, CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint32_t box_inner, uint32_t box_outer) {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    KBO_CUDA(h, cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
    if (q != cudaDriverEntryPointSuccess || !p) KBO_FAIL(h, KBO_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    fn = (PFN_encodeTiled)p;
  }
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {inner * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) KBO_FAIL(h, KBO_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return KBO_OK;
}

int kbo_i_tc_variance(kbo_handle* h, const __half* Ksh, const __half* Ksl, int64_t rows, const __half* Wh, const __half* Wl, int Npad,
                      double /*unused*/, double amp, float* var_n_out, int k_span, cudaStream_t s, int nprod, int jtiles) {
  return tc_launch(h, Ksh, Ksl, rows, Wh, Wl, Npad, h->scal.p + S_WSCALE, amp, var_n_out, nullptr, k_span, s, nprod, jtiles);
}

// Raw entry for the kernel-level parity test: caller supplies fp16 planes and the scale pair on the device.
extern "C" int kbo_tc_variance_raw(kbo_handle* h, const void* Ksh, const void* Ksl, int64_t rows, const void* Wh, const void* Wl, int32_t Npad,
                                   const double* w_scale_dev, double amp, float* var_out, double* sumsq_out, int32_t k_span, void* stream) {
  if (!h) return KBO_ERR_INVALID;
  return tc_launch(h, (const __half*)Ksh, (const __half*)Ksl, rows, (const __half*)Wh, (const __half*)Wl, Npad, w_scale_dev, amp, var_out,
                   sumsq_out, k_span, (cudaStream_t)stream);
}
