// GEMM v2 for sm_90a: persistent, stream-K balanced wgmma GEMM / implicit-GEMM conv3x3.
//
//   out[M, N] = epilogue( A[M, K] . W[N, K]^T )        fp16 operands, fp32 accumulation in registers
//
// Replaces (reference file:line): attention.py:41,62,121-125,175-179,297,354,363;
// openaimodel.py:109,134,186,205,213,361-363,464; text_grounding_net.py:75-81; convnext.py:30-32,71-81.
// Design points:
//   * one persistent CTA per SM; work = (128 x BN tile, k-block range) segments.  Full waves of
//     tiles are processed data-parallel; the ragged last 1-2 waves are split evenly over all CTAs
//     in units of 64-wide k-blocks ("stream-K"), so 40-, 160- and 320-tile problems do not leave
//     most SMs idle.  A tile shared by several CTAs is finished by the CTA that holds its first
//     k-blocks; the others publish fp32 partials (coalesced, L2-resident) and a per-warp flag, and
//     the owner adds them in a fixed order -> bit-reproducible.
//   * BN in {128, 160, 192, 256} chosen per N (320 = 2 x 160, 960 = 5 x 192, 1280 = 5 x 256 ...):
//     no padded columns, half the A-tile traffic of 128-wide tiles.
//   * warp roles (384 threads = 3 warpgroups): warpgroup 0 holds the TMA producer (warp 0, one thread)
//     and the epilogue store warp (warp 1, one thread); the group gives its registers to the consumers
//     with setmaxnreg.  Warpgroups 1 and 2 are consumers that own 64 rows of the tile each: wgmma
//     m64nBNk16 from the 128B-swizzled operand ring into register accumulators, then the fused epilogue.
//     The producer runs ahead across segments, so the next tile's operands land during the epilogue.
//   * staged epilogue (16-bit outputs): one tile-sized buffer in shared memory, in 32-column slabs of
//     128 rows x 64 B (64B swizzle).  The store warp TMA-loads the tile's residual into it while the
//     consumers run the mainloop; the consumers read it with ldmatrix in accumulator-fragment order,
//     write the packed result back in place with stmatrix and go straight on to the next tile's
//     mainloop; the store warp writes the buffer out with TMA stores (rows past M / past the conv
//     image, columns past N clipped by the tensor map) and reloads it for the next tile once the
//     stores have read it.  Only the final conv's fp32 NCHW output is stored from the fragments.
// conv3x3 gathers the A tile tap by tap with a 4-D TMA box over the NHWC activation; out-of-image taps
// are zero-filled by the TMA unit (no im2col buffer, no halo copy).
#include "../../include/idiff_b200.h"
#include "common.cuh"
#include "host.cuh"
#include "wgmma.cuh"

#include <stdlib.h>

namespace idiff {
namespace v2 {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;
constexpr int THREADS = 384;
constexpr int CONSUMER_WARPS = 8;  // stream-K publish flags per CTA: one per consumer warp

struct Params {
  int M, N, K, KB;
  int n_tiles, T, T_dp, G;
  long U_sk;  // stream-K units (k-blocks) = (T - T_dp) * KB
  // conv geometry
  int conv, H, W, Bn, PW, PH, PB, tiles_w, tiles_h, kb_per_tap;
  // epilogue
  const float* bias;
  const h16* rowadd;
  const h16* residual;
  void* out;
  int ldo, ldr, ldra, rows_per_batch, flags;
  float gate;
  const float* gate_b;  // optional per-batch-entry factor of the residual gate (header: gate_b)
  // stream-K fixup
  float* ws;    // [G][BN/8][256 consumer threads][4] fp32 partial tiles, in accumulator-fragment order
  int* sflags;  // [G][CONSUMER_WARPS] publish flags (fixed location, self-resetting)
  unsigned long long* trace;  // optional [G][16] %globaltimer stamps (idiff_set_gemm_trace), else null
  // LayerNorm folded across GEMMs (header: ln_* fields)
  float2* ln_out;        // producer: [n_tiles][M] partial (sum, sumsq) of the output rows
  const float2* ln_in;   // consumer: [ln_slots][M] partials of the A rows
  const float* ln_s;     // consumer: [N] column sums of the gamma-folded fp16 weights
  int ln_slots;
  float ln_eps;
};

constexpr int MODE_PLAIN = 0;  // bias / row-add, optional SiLU / GELU, optional gate*x + residual, fp16 out
constexpr int MODE_GEGLU = 1;  // (value + b) * gelu(gate + b), fp16 out with N/2 columns
constexpr int MODE_NCHW = 2;   // fp32 (B, N, HW) output (the final conv -> eps)
constexpr int MODE_GATED = 3;  // bias, gate * gate_b[batch entry] * x + residual, fp16 out (per-image fuser scales)

constexpr int EPI_SLAB_COLS = 32;                        // columns of one epilogue slab / TMA box (64 B rows)
constexpr int EPI_SLAB_BYTES = BM * EPI_SLAB_COLS * 2;   // 8 KB

template <int BN, int MODE>
struct Cfg {
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  // epilogue buffer: the 128 x EW output tile (GEGLU: BN/2 columns; none for the fp32 NCHW output)
  static constexpr int EW = MODE == MODE_NCHW ? 0 : MODE == MODE_GEGLU ? BN / 2 : BN;
  static constexpr int EPI_BYTES = BM * EW * 2;
  static constexpr int BAR_BYTES = 256;          // 2 * STAGES + 2 mbarriers
  static constexpr int FIXED = 1024 + BAR_BYTES;  // + slack to align the ring to 1024 B (SWIZZLE_128B)
  static constexpr int STAGES_FIT = (227 * 1024 - FIXED - EPI_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > 6 ? 6 : STAGES_FIT;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + FIXED;
  static constexpr int ACC = BN / 2;  // fp32 accumulator registers per consumer thread (64 x BN per warpgroup)
  static_assert(STAGES >= 3, "operand ring too shallow");
  static_assert(EW % EPI_SLAB_COLS == 0, "epilogue slabs must tile the output columns exactly");
  static_assert(STAGE_BYTES % 1024 == 0, "the epilogue buffer after the ring must stay 1024 B aligned");
};

struct Seg {
  int tile, kb0, kb1;
};

// Work iterator shared by the roles: stream-K range first, then data-parallel tiles.
struct WorkIter {
  const Params& p;
  int cta;
  long u, u1;  // stream-K cursor / end (units)
  int dp_next;
  __device__ WorkIter(const Params& p_, int cta_) : p(p_), cta(cta_) {
    u = (p.U_sk * cta) / p.G;
    u1 = (p.U_sk * (cta + 1)) / p.G;
    dp_next = cta;
  }
  __device__ bool next(Seg& s) {
    if (u < u1) {
      const int t_local = (int)(u / p.KB);
      const int kb0 = (int)(u - (long)t_local * p.KB);
      const long rem = u1 - u;
      const int kb1 = (rem < (long)(p.KB - kb0)) ? (int)(kb0 + rem) : p.KB;
      s.tile = p.T_dp + t_local;
      s.kb0 = kb0;
      s.kb1 = kb1;
      u += kb1 - kb0;
      return true;
    }
    if (dp_next < p.T_dp) {
      s.tile = dp_next;
      s.kb0 = 0;
      s.kb1 = p.KB;
      dp_next += p.G;
      return true;
    }
    return false;
  }
};

IDIFF_DEVICE int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
  return v;
}
IDIFF_DEVICE void st_release_gpu(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;\n" ::"l"(p), "r"(v) : "memory");
}
IDIFF_DEVICE float2 ld_pair(const h16* p) { return unpack_half2(*reinterpret_cast<const uint32_t*>(p)); }

// Byte offset in the epilogue buffer of the 16 B chunk holding tile row `row`, columns [8 jj, 8 jj + 8):
// 32-column slabs of 128 rows x 64 B, each row's four chunks permuted as the TMA unit's 64B swizzle does
// (chunk ^= (row / 2) % 4), so the 8 rows of one ldmatrix / stmatrix phase hit 8 different 16 B bank groups.
IDIFF_DEVICE uint32_t epi_offset(int row, int jj) {
  return (uint32_t)((jj >> 2) * EPI_SLAB_BYTES + row * 64 + (((jj & 3) ^ ((row >> 1) & 3)) << 4));
}

template <int BN, int MODE>
__global__ void __launch_bounds__(THREADS, 1)
gemm2_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
             const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmR, const Params p) {
  using C = Cfg<BN, MODE>;
  constexpr int STAGES = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_STAGE_BYTES;
  uint8_t* sE = smem + STAGES * C::STAGE_BYTES;  // epilogue buffer (C::EPI_BYTES)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sE + C::EPI_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* epi_ready = empty_bar + STAGES;  // the tile's residual has landed in sE (or: sE is free, no residual)
  uint64_t* epi_full = epi_ready + 1;        // the consumers have staged the tile's output in sE

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int cta = blockIdx.x;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (C::EW > 0) {
      tma_prefetch_desc(&tmO);
      if (p.residual) tma_prefetch_desc(&tmR);
    }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], CONSUMER_WARPS);  // one arrival per consumer warp
    }
    mbar_init(epi_ready, 1);
    mbar_init(epi_full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();  // the next kernel's prologue may overlap this kernel (host.cuh launch_pdl)
  pdl_wait();               // operands come from earlier kernels: nothing above touched global memory
  auto stamp = [&](int slot) {
    if (p.trace) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      p.trace[(long)blockIdx.x * 16 + slot] = t;
    }
  };
  // a phase of the CTA's first and of its last epilogue tile: slot (kept once written) and slot + 3
  auto stamp_tile = [&](int slot) {
    if (p.trace) {
      if (p.trace[(long)blockIdx.x * 16 + slot] == 0) stamp(slot);
      stamp(slot + 3);
    }
  };
  if (threadIdx.x == 0) {
    stamp(0);
    if (p.trace) p.trace[(long)blockIdx.x * 16 + 12] = (unsigned long long)clock64();  // SM clock at entry
  }

  auto tile_origin = [&](int tile, int& n0, int& m0, int& b0, int& h0, int& w0) {
    const int n_tile = tile % p.n_tiles;
    const int m_tile = tile / p.n_tiles;
    n0 = n_tile * BN;
    m0 = m_tile * BM;
    b0 = h0 = w0 = 0;
    if (p.conv) {
      const int tw = m_tile % p.tiles_w;
      const int th = (m_tile / p.tiles_w) % p.tiles_h;
      const int tb = m_tile / (p.tiles_w * p.tiles_h);
      b0 = tb * p.PB;
      h0 = th * p.PH;
      w0 = tw * p.PW;
    }
  };

  // Register split (setmaxnreg at the head of each role branch): 40 x 128 + 232 x 256 <= the CTA's 65536.
  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n");
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      WorkIter it(p, cta);
      Seg sg;
      uint32_t s = 0, ph = 0;  // ring position: running stage / phase
      while (it.next(sg)) {
        int n0, m0, b0, h0, w0;
        tile_origin(sg.tile, n0, m0, b0, h0, w0);
        // conv: k-block kb = (tap, 64-channel slice cb); walked incrementally
        int tap = 0, cb = 0, ky = 0, kx = 0;
        if (p.conv) {
          tap = sg.kb0 / p.kb_per_tap;
          cb = sg.kb0 - tap * p.kb_per_tap;
          ky = tap / 3;
          kx = tap - ky * 3;
        }
        for (int kb = sg.kb0; kb < sg.kb1; ++kb) {
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_expect_tx(&full_bar[s], C::STAGE_BYTES);
          if (p.conv) {
            tma_load_4d(sA + s * A_STAGE_BYTES, &tmA, &full_bar[s], cb * BK, w0 + kx - 1, h0 + ky - 1, b0);
            if (++cb == p.kb_per_tap) {
              cb = 0;
              if (++kx == 3) {
                kx = 0;
                ++ky;
              }
            }
          } else {
            tma_load_2d(sA + s * A_STAGE_BYTES, &tmA, &full_bar[s], kb * BK, m0);
          }
          tma_load_2d(sB + s * C::B_STAGE_BYTES, &tmB, &full_bar[s], kb * BK, n0);
          if (++s == STAGES) {
            s = 0;
            ph ^= 1;
          }
        }
      }
    } else if (C::EW > 0 && warp == 1 && lane == 0) {
      // ===================== epilogue store warp: residual in, result out =====================
      // Per owner segment (the ones that run an epilogue): fill sE with the tile's residual (or just
      // release it to the consumers), wait until they have staged the result there, store it, and wait
      // until the stores have read sE before the next tile's residual may overwrite it.
      WorkIter it(p, cta);
      Seg sg;
      uint32_t ep = 0;
      const int n_out = MODE == MODE_GEGLU ? p.N / 2 : p.N;
      while (it.next(sg)) {
        if (sg.kb0 != 0) continue;
        int n0, m0, b0, h0, w0;
        tile_origin(sg.tile, n0, m0, b0, h0, w0);
        const int oc0 = MODE == MODE_GEGLU ? (sg.tile % p.n_tiles) * (BN / 2) : n0;
        const int rem = (n_out - oc0 + EPI_SLAB_COLS - 1) / EPI_SLAB_COLS;  // slabs not wholly past N
        const int slabs = rem < C::EW / EPI_SLAB_COLS ? rem : C::EW / EPI_SLAB_COLS;
        if (p.residual) {
          mbar_expect_tx(epi_ready, slabs * EPI_SLAB_BYTES);  // clipped box elements count (zero-filled)
          for (int q = 0; q < slabs; ++q) {
            if (p.conv) tma_load_4d(sE + q * EPI_SLAB_BYTES, &tmR, epi_ready, oc0 + q * EPI_SLAB_COLS, w0, h0, b0);
            else tma_load_2d(sE + q * EPI_SLAB_BYTES, &tmR, epi_ready, oc0 + q * EPI_SLAB_COLS, m0);
          }
        } else {
          mbar_arrive(epi_ready);
        }
        mbar_wait(epi_full, ep);
        ep ^= 1;
        for (int q = 0; q < slabs; ++q) {
          if (p.conv) tma_store_4d(&tmO, sE + q * EPI_SLAB_BYTES, oc0 + q * EPI_SLAB_COLS, w0, h0, b0);
          else tma_store_2d(&tmO, sE + q * EPI_SLAB_BYTES, oc0 + q * EPI_SLAB_COLS, m0);
        }
        tma_store_commit();
        stamp_tile(3);
        tma_store_wait_read();
      }
      tma_store_wait_all();
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n");
    // ===================== consumers: mainloop + epilogue =====================
    const int cw = (warp >> 2) - 1;  // consumer warpgroup: tile rows [64 cw, 64 cw + 64)
    const int ew = warp - 4;         // consumer warp 0..7
    const int ct = threadIdx.x - 128;  // consumer thread 0..255
    const int t4 = lane & 3;
    // tile rows of this thread (accumulator fragment: wgmma.cuh): rl0 and rl0 + 8
    const int rl0 = cw * 64 + (warp & 3) * 16 + (lane >> 2);
    constexpr bool geglu = (MODE == MODE_GEGLU);
    constexpr bool nchw = (MODE == MODE_NCHW);
    constexpr bool gated = (MODE == MODE_GATED);
    constexpr int NJ = BN / 8;                     // 8-column groups of the accumulator
    constexpr int NJO = geglu ? NJ / 2 : NJ;       // ... that produce output columns
    const bool do_silu = !gated && (p.flags & IDIFF_EPI_SILU) != 0;
    const bool do_gelu = !gated && (p.flags & IDIFF_EPI_GELU) != 0;
    const int n_out_total = geglu ? p.N / 2 : p.N;
    // K-major SWIZZLE_128B descriptors of stage 0; a stage / 16-deep k-step is an address offset (>> 4)
    const uint64_t da0 = make_wgmma_desc(smem_u32(sA) + cw * 64 * 128, 16, 1024);
    const uint64_t db0 = make_wgmma_desc(smem_u32(sB), 16, 1024);

    float acc[C::ACC];
    WorkIter it(p, cta);
    Seg sg;
    uint32_t s = 0, ph = 0;
    uint32_t ep = 0;  // epilogue buffer phase
    while (it.next(sg)) {
      int n0, m0, b0, h0, w0;
      tile_origin(sg.tile, n0, m0, b0, h0, w0);
      // ---- mainloop: one k-block of wgmmas in flight while the next stage's barrier is awaited ----
      uint32_t prev = 0;
      for (int kb = sg.kb0; kb < sg.kb1; ++kb) {
        mbar_wait(&full_bar[s], ph);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          Wgmma<BN>::ss(acc, da0 + ((s * A_STAGE_BYTES + k * 32) >> 4), db0 + ((s * C::B_STAGE_BYTES + k * 32) >> 4),
                        (kb > sg.kb0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's wgmmas have finished reading their stage
        if (kb > sg.kb0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = s;
        if (++s == STAGES) {
          s = 0;
          ph ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (lane == 0) mbar_arrive(&empty_bar[prev]);

      const bool owner = sg.kb0 == 0;
      if (owner && ct == 0) stamp_tile(1);
      const bool complete = owner && sg.kb1 == p.KB;
      const bool fixup = owner && !complete;  // this CTA holds the tile's first k-blocks, others the rest
      const long fstride = (long)BM * BN / 4;  // float4s of one CTA's partial tile
      if (!owner) {
        // ---- publish the fp32 partial in fragment order: ws[cta][i][consumer thread] (coalesced float4s) ----
        float4* dst = reinterpret_cast<float4*>(p.ws) + (long)cta * fstride + ct;
#pragma unroll
        for (int i = 0; i < C::ACC / 4; ++i)
          __stcg(dst + i * 256, make_float4(acc[4 * i], acc[4 * i + 1], acc[4 * i + 2], acc[4 * i + 3]));
        __threadfence();
        __syncwarp();
        if (lane == 0) st_release_gpu(p.sflags + cta * CONSUMER_WARPS + ew, 1);
        continue;
      }
      // followers of an incomplete owner segment: the CTAs covering the tile's remaining k-blocks
      int f0 = 0, f1 = -1;
      if (fixup) {
        const long tile_u0 = (long)(sg.tile - p.T_dp) * p.KB;
        f0 = (int)(((tile_u0 + sg.kb1 + 1) * p.G + p.U_sk - 1) / p.U_sk) - 1;
        f1 = (int)(((tile_u0 + p.KB) * p.G + p.U_sk - 1) / p.U_sk) - 1;
        for (int f = f0; f <= f1; ++f) {
          const int* fl = p.sflags + f * CONSUMER_WARPS + ew;
          const long long t0 = clock64();
          while (ld_acquire_gpu(fl) == 0) {
            if (clock64() - t0 > 8000000000LL) __trap();  // bounded: a schedule bug traps instead of hanging
          }
        }
        // the followers' partials in CTA order (bit-reproducible)
        for (int f = f0; f <= f1; ++f) {
          const float4* src = reinterpret_cast<const float4*>(p.ws) + (long)f * fstride + ct;
#pragma unroll
          for (int i = 0; i < C::ACC / 4; ++i) {
            const float4 v = __ldcg(src + i * 256);
            acc[4 * i] += v.x;
            acc[4 * i + 1] += v.y;
            acc[4 * i + 2] += v.z;
            acc[4 * i + 3] += v.w;
          }
        }
        // consume the followers' flags so the next launch (or graph replay) starts clean
        __syncwarp();
        if (lane == 0)
          for (int f = f0; f <= f1; ++f) st_release_gpu(p.sflags + f * CONSUMER_WARPS + ew, 0);
      }

      // ---- fused epilogue: rows rl0 / rl0 + 8, column pairs 8j + 2 t4 ----
      long orow[2];
      bool rok[2];
      int bidx[2], pix[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int rl = rl0 + 8 * hh;
        if (p.conv) {
          const int pw = rl % p.PW;
          const int ph_ = (rl / p.PW) % p.PH;
          const int pb = rl / (p.PW * p.PH);
          const int b = b0 + pb, h = h0 + ph_, w = w0 + pw;
          rok[hh] = (b < p.Bn) && (h < p.H) && (w < p.W);
          pix[hh] = h * p.W + w;
          orow[hh] = (long)b * p.H * p.W + pix[hh];
          bidx[hh] = b;
        } else {
          orow[hh] = (long)m0 + rl;
          rok[hh] = orow[hh] < p.M;
          bidx[hh] = (int)(orow[hh] / p.rows_per_batch);
          pix[hh] = (int)(orow[hh] - (long)bidx[hh] * p.rows_per_batch);
        }
      }
      // LayerNorm fold, consumer side: each row's mean / rstd from the producer GEMM's partial sums, added in
      // slot order (deterministic).  y = rstd * (x . W'^T - mean * colsum(W')) + (W beta + b).
      const bool lni = !gated && p.ln_in != nullptr;
      float ln_rstd[2] = {1.f, 1.f}, ln_nmean[2] = {0.f, 0.f};
      if (lni) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          float a = 0.f, q = 0.f;
          if (rok[hh]) {
            for (int sl = 0; sl < p.ln_slots; ++sl) {
              const float2 v = __ldcg(p.ln_in + (long)sl * p.M + orow[hh]);
              a += v.x;
              q += v.y;
            }
          }
          const float inv_k = 1.0f / (float)p.K;
          const float mean = a * inv_k;
          ln_rstd[hh] = rsqrtf(fmaxf(q * inv_k - mean * mean, 0.f) + p.ln_eps);
          ln_nmean[hh] = -mean * ln_rstd[hh];
        }
      }
      const int out_col_base = geglu ? (sg.tile % p.n_tiles) * (BN / 2) : n0;
      const bool has_res = p.residual != nullptr;
      const bool lno = p.ln_out != nullptr;
      float ln_ps[2] = {0.f, 0.f}, ln_pq[2] = {0.f, 0.f};
      const float gate = p.gate;
      // MODE_GATED: the residual gate of each row is gate * gate_b[its batch entry]
      float gate_r[2] = {gate, gate};
      if (gated) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
          if (rok[hh]) gate_r[hh] = gate * __ldg(p.gate_b + bidx[hh]);
      }
      // column vectors of the 8-column group j at this thread's column pair (zero for columns past N)
      auto col_vecs = [&](int j, float2& bv, float2& bg, float2& sv, float2& sgt) {
        const int c = 8 * j + 2 * t4;  // tile column of the pair (GEGLU: value column; its gate is BN/2 further on)
        const int oc = out_col_base + c;
        bv = bg = sv = sgt = make_float2(0.f, 0.f);
        if (oc >= n_out_total) return;  // 16-bit outputs have N % 8 == 0: a pair is wholly inside or outside
        const bool hi = !nchw || oc + 1 < n_out_total;  // fp32 NCHW output may have an odd N (the final conv: 3 or 4)
        if (p.bias) {
          if (nchw) bv = make_float2(__ldg(p.bias + n0 + c), hi ? __ldg(p.bias + n0 + c + 1) : 0.f);
          else bv = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + c));
          if (geglu) bg = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + BN / 2 + c));
        }
        if (lni) {
          sv = __ldg(reinterpret_cast<const float2*>(p.ln_s + n0 + c));
          if (geglu) sgt = __ldg(reinterpret_cast<const float2*>(p.ln_s + n0 + BN / 2 + c));
        }
      };
      // bias or LayerNorm fold, then GEGLU, or row-add and SiLU / GELU, of the pair (j, row half hh)
      auto act_pair = [&](int j, int hh, const float2& bv, const float2& bg, const float2& sv, const float2& sgt,
                          float& x0, float& x1) {
        x0 = acc[4 * j + 2 * hh];
        x1 = acc[4 * j + 2 * hh + 1];
        if (lni) {
          x0 = fmaf(ln_rstd[hh], x0, fmaf(ln_nmean[hh], sv.x, bv.x));
          x1 = fmaf(ln_rstd[hh], x1, fmaf(ln_nmean[hh], sv.y, bv.y));
        } else {
          x0 += bv.x;
          x1 += bv.y;
        }
        if (geglu) {
          float g0 = acc[4 * (j + NJ / 2) + 2 * hh], g1 = acc[4 * (j + NJ / 2) + 2 * hh + 1];
          if (lni) {
            g0 = fmaf(ln_rstd[hh], g0, fmaf(ln_nmean[hh], sgt.x, bg.x));
            g1 = fmaf(ln_rstd[hh], g1, fmaf(ln_nmean[hh], sgt.y, bg.y));
          } else {
            g0 += bg.x;
            g1 += bg.y;
          }
          x0 *= gelu_erf_f(g0);
          x1 *= gelu_erf_f(g1);
        } else {
          if (!gated && p.rowadd && rok[hh] && out_col_base + 8 * j < n_out_total) {
            const float2 f = ld_pair(p.rowadd + (long)bidx[hh] * p.ldra + n0 + 8 * j + 2 * t4);
            x0 += f.x;
            x1 += f.y;
          }
          if (do_silu) {
            x0 = silu_f(x0);
            x1 = silu_f(x1);
          } else if (do_gelu) {
            x0 = gelu_erf_f(x0);
            x1 = gelu_erf_f(x1);
          }
        }
      };
      if constexpr (nchw) {
        // fp32 NCHW (the final conv, one launch per forward): stored straight from the fragments
        float* o = reinterpret_cast<float*>(p.out);
        const long hw = p.conv ? (long)p.H * p.W : (long)p.rows_per_batch;
#pragma unroll
        for (int j = 0; j < NJO; ++j) {
          const int oc = out_col_base + 8 * j + 2 * t4;
          if (oc >= n_out_total) continue;
          float2 bv, bg, sv, sgt;
          col_vecs(j, bv, bg, sv, sgt);
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            if (!rok[hh]) continue;
            float x0, x1;
            act_pair(j, hh, bv, bg, sv, sgt, x0, x1);
            o[((long)bidx[hh] * n_out_total + oc) * hw + pix[hh]] = x0;
            if (oc + 1 < n_out_total) o[((long)bidx[hh] * n_out_total + oc + 1) * hw + pix[hh]] = x1;
          }
        }
      } else {
        // 16-bit output, staged in sE: one ldmatrix / stmatrix x4 covers the groups j = 2 jp, 2 jp + 1 of both row
        // halves (matrix 2u + hh = group 2 jp + u, rows 8 hh ..); lane l gives the address of row l % 8 of matrix l / 8.
        // Rows past M / past the conv image and columns past N are computed on whatever sE holds and clipped by
        // the TMA store.
        const int lrow = cw * 64 + (warp & 3) * 16 + 8 * ((lane >> 3) & 1) + (lane & 7);
        const uint32_t se = smem_u32(sE);
        mbar_wait(epi_ready, ep);
        ep ^= 1;
#pragma unroll
        for (int jp = 0; jp < NJO / 2; ++jp) {
          const uint32_t addr = se + epi_offset(lrow, 2 * jp + (lane >> 4));
          uint32_t rr[4] = {0u, 0u, 0u, 0u};
          if (has_res) ldmatrix_x4(rr, addr);
          uint32_t packed[4];
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int j = 2 * jp + u;
            const bool cok = out_col_base + 8 * j < n_out_total;
            float2 bv, bg, sv, sgt;
            col_vecs(j, bv, bg, sv, sgt);
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              float x0, x1;
              act_pair(j, hh, bv, bg, sv, sgt, x0, x1);
              if (has_res) {
                const float2 r = unpack_half2(rr[2 * u + hh]);
                const float g = gated ? gate_r[hh] : gate;
                x0 = fmaf(g, x0, r.x);
                x1 = fmaf(g, x1, r.y);
              }
              if (lno && cok) {
                ln_ps[hh] += x0 + x1;
                ln_pq[hh] = fmaf(x0, x0, fmaf(x1, x1, ln_pq[hh]));
              }
              packed[2 * u + hh] = pack_half2(x0, x1);
            }
          }
          stmatrix_x4(addr, packed);
        }
        fence_proxy_async_smem();  // the stmatrix writes -> visible to the TMA store
        named_bar_sync(1, 256);
        if (ct == 0) {
          mbar_arrive(epi_full);
          stamp_tile(2);
        }
      }
      // LayerNorm fold, producer side: the row's (sum, sumsq) over this tile's columns, slot = n tile
      if (lno) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          float a = ln_ps[hh], q = ln_pq[hh];
          a += __shfl_xor_sync(0xffffffffu, a, 1);
          q += __shfl_xor_sync(0xffffffffu, q, 1);
          a += __shfl_xor_sync(0xffffffffu, a, 2);
          q += __shfl_xor_sync(0xffffffffu, q, 2);
          if (t4 == 0 && rok[hh]) __stcg(p.ln_out + (long)(sg.tile % p.n_tiles) * p.M + orow[hh], make_float2(a, q));
        }
      }
    }
  }

  __syncthreads();
  if (threadIdx.x == 0) {
    stamp(7);
    if (p.trace) p.trace[(long)blockIdx.x * 16 + 13] = (unsigned long long)clock64();  // SM clock at exit
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static void* g_ws = nullptr;
static unsigned long long* g_trace = nullptr;
static long g_ws_bytes = 0;
static int g_num_sms = 0;
constexpr long kFlagBytes = 64 * 1024;

static void choose_patch(int H, int W, int* PW, int* PH, int* PB) {
  int pw = 1;
  while (pw * 2 <= 128 && (W % (pw * 2)) == 0) pw *= 2;
  int ph = 1;
  while (pw * ph * 2 <= 128 && ph < H) ph *= 2;
  *PW = pw;
  *PH = ph;
  *PB = 128 / (pw * ph);
}

// Tensor map of a 16-bit epilogue operand (the output, or the residual) with `n` columns and row stride `ld`
// elements, in boxes of one epilogue slab: (32 columns, 128 rows) for a linear layer, (32, PW, PH, PB) over
// the NHWC image for conv3x3 -- the rows of the tile's A patch.  Its bounds clip the boxes of edge tiles.
static int encode_epi_map(CUtensorMap* m, const void* base, int n, int ld, const idiff_gemm_args* a, const Params& p) {
  if (p.conv) {
    const uint64_t dims[4] = {(uint64_t)n, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.Bn};
    const uint64_t strides[3] = {(uint64_t)ld * 2, (uint64_t)p.W * ld * 2, (uint64_t)p.H * p.W * ld * 2};
    const uint32_t box[4] = {(uint32_t)EPI_SLAB_COLS, (uint32_t)p.PW, (uint32_t)p.PH, (uint32_t)p.PB};
    return encode_tmap_f16_sw(m, base, 4, dims, strides, box, 64);
  }
  const uint64_t dims[2] = {(uint64_t)n, (uint64_t)a->M};
  const uint64_t strides[1] = {(uint64_t)ld * 2};
  const uint32_t box[2] = {(uint32_t)EPI_SLAB_COLS, (uint32_t)BM};
  return encode_tmap_f16_sw(m, base, 2, dims, strides, box, 64);
}

template <int BN, int MODE>
static int launch(const idiff_gemm_args* a, cudaStream_t stream, bool want_sk) {
  using C = Cfg<BN, MODE>;
  Params p;
  memset(&p, 0, sizeof(p));
  p.M = a->M;
  p.N = a->N;
  p.K = a->K;
  p.KB = (a->K + BK - 1) / BK;
  p.bias = a->bias;
  p.rowadd = reinterpret_cast<const h16*>(a->rowadd);
  p.residual = reinterpret_cast<const h16*>(a->residual);
  p.out = a->out;
  p.ldo = a->ldo;
  p.ldr = a->ldr;
  p.ldra = a->ldra > 0 ? a->ldra : a->N;
  p.rows_per_batch = a->rows_per_batch > 0 ? a->rows_per_batch : a->M;
  p.flags = a->flags;
  p.gate = a->gate;
  p.gate_b = a->gate_b;
  p.trace = g_trace;
  p.ln_out = reinterpret_cast<float2*>(a->ln_stats_out);
  p.ln_in = reinterpret_cast<const float2*>(a->ln_stats_in);
  p.ln_s = a->ln_colsum;
  p.ln_slots = a->ln_slots_in;
  p.ln_eps = a->ln_eps;

  CUtensorMap tmA, tmB;
  int m_tiles;
  if (a->conv_h > 0) {
    const int H = a->conv_h, W = a->conv_w, B = a->conv_b, Cn = a->conv_cin;
    IDIFF_REQUIRE(Cn % BK == 0, "conv3x3: Cin=%d must be a multiple of %d", Cn, BK);
    IDIFF_REQUIRE(a->K == 9 * Cn, "conv3x3: K=%d must equal 9*Cin=%d", a->K, 9 * Cn);
    IDIFF_REQUIRE(a->M == B * H * W, "conv3x3: M=%d must equal B*H*W=%d", a->M, B * H * W);
    p.conv = 1;
    p.H = H;
    p.W = W;
    p.Bn = B;
    choose_patch(H, W, &p.PW, &p.PH, &p.PB);
    p.tiles_w = W / p.PW;
    p.tiles_h = (H + p.PH - 1) / p.PH;
    const int tiles_b = (B + p.PB - 1) / p.PB;
    p.kb_per_tap = Cn / BK;
    p.rows_per_batch = H * W;
    m_tiles = p.tiles_w * p.tiles_h * tiles_b;
    const uint64_t dims[4] = {(uint64_t)Cn, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    const uint64_t strides[3] = {(uint64_t)Cn * 2, (uint64_t)W * Cn * 2, (uint64_t)H * W * Cn * 2};
    const uint32_t box[4] = {(uint32_t)BK, (uint32_t)p.PW, (uint32_t)p.PH, (uint32_t)p.PB};
    if (encode_tmap_f16(&tmA, a->a, 4, dims, strides, box)) return -1;
  } else {
    m_tiles = (a->M + BM - 1) / BM;
    const uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->M};
    const uint64_t strides[1] = {(uint64_t)a->lda * 2};
    const uint32_t box[2] = {(uint32_t)BK, (uint32_t)BM};
    if (encode_tmap_f16(&tmA, a->a, 2, dims, strides, box)) return -1;
  }
  {
    const uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->N};
    const uint64_t strides[1] = {(uint64_t)a->ldw * 2};
    const uint32_t box[2] = {(uint32_t)BK, (uint32_t)BN};
    if (encode_tmap_f16(&tmB, a->w, 2, dims, strides, box)) return -1;
  }
  p.n_tiles = (a->N + BN - 1) / BN;
  p.T = p.n_tiles * m_tiles;
  CUtensorMap tmO, tmR;
  memset(&tmO, 0, sizeof(tmO));
  memset(&tmR, 0, sizeof(tmR));
  if (C::EW > 0) {
    if (encode_epi_map(&tmO, a->out, MODE == MODE_GEGLU ? a->N / 2 : a->N, a->ldo, a, p)) return -1;
    if (a->residual && encode_epi_map(&tmR, a->residual, a->N, a->ldr, a, p)) return -1;
  }

  if (g_num_sms == 0) {
    int dev = 0;
    IDIFF_CHECK_CUDA(cudaGetDevice(&dev));
    IDIFF_CHECK_CUDA(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  // Stream-K needs the fixup workspace (flags in its first 64 KiB, partial tiles after); short-K
  // problems (fixup cost ~ mainloop) and exact multiples of the SM count stay data-parallel.
  const long ws_need = kFlagBytes + (long)g_num_sms * 128 * BN * sizeof(float);
  // per-call scratch (idiff_gemm_args.workspace: one per stream, so concurrent streams never share flags)
  // takes precedence over the process-wide default of idiff_set_gemm_workspace
  void* ws_ptr = a->workspace ? a->workspace : g_ws;
  const long ws_bytes = a->workspace ? a->workspace_bytes : g_ws_bytes;
  const int workers = g_num_sms;
  const bool use_sk = want_sk && ws_ptr && ws_bytes >= ws_need && p.KB >= 8 && (p.T % g_num_sms) != 0 &&
                      (long)p.T * p.KB >= g_num_sms;
  if (use_sk) {
    p.G = g_num_sms;
    const int waves = p.T / p.G;
    p.T_dp = (waves >= 2) ? (waves - 1) * p.G : 0;
    p.U_sk = (long)(p.T - p.T_dp) * p.KB;
    p.sflags = reinterpret_cast<int*>(ws_ptr);
    p.ws = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ws_ptr) + kFlagBytes);
  } else {
    p.G = workers < p.T ? workers : p.T;
    p.T_dp = p.T;
    p.U_sk = 0;
  }

  static bool attr_set = false;
  if (!attr_set) {
    IDIFF_CHECK_CUDA(cudaFuncSetAttribute(gemm2_kernel<BN, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          C::SMEM_BYTES));
    attr_set = true;
  }
  IDIFF_CHECK_CUDA(launch_pdl(gemm2_kernel<BN, MODE>, dim3(p.G), dim3(THREADS), C::SMEM_BYTES, stream, tmA, tmB, tmO, tmR, p));
  IDIFF_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// Tile width and schedule.  A small cost model in SM clocks (its constants are estimates, not fitted to H100
// measurements; tools/plan_sweep.py sweeps the alternatives):
//   * one 64-deep k-block of a 128 x BN tile costs max(tensor time 2*BN, operand bytes / ~80 B/clk/SM);
//   * data-parallel: ceil(T / SMs) rounds of (KB k-blocks + ~600 clk of pipeline fill) and one exposed
//     epilogue;
//   * stream-K: the k-blocks of the last partial round are spread evenly, but the fixup costs a fixed
//     ~20k clk of flag / partial-tile round trips plus the owner pulling every follower's fp32 tile
//     through one SM's L2 port (~40 B/clk), so it only pays for long-K tiles.
struct Plan {
  int bn;
  bool sk;
};
static int count_m_tiles(const idiff_gemm_args* a) {
  if (a->conv_h > 0) {
    int pw, ph, pb;
    choose_patch(a->conv_h, a->conv_w, &pw, &ph, &pb);
    return (a->conv_w / pw) * ((a->conv_h + ph - 1) / ph) * ((a->conv_b + pb - 1) / pb);
  }
  return (a->M + BM - 1) / BM;
}
// fixed_bn: 0 = choose the tile width, at most max_bn
static Plan plan_gemm(const idiff_gemm_args* a, int fixed_bn, int max_bn = 256) {
  const char* force = getenv("IDIFF_GEMM_PLAN");  // "bn,sk" overrides the model (tests, tuning); bn 0 = keep
  if (g_num_sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  const int sms = g_num_sms;
  const int KB = (a->K + BK - 1) / BK;
  const int m_tiles = count_m_tiles(a);
  const int cands[4] = {256, 192, 160, 128};
  long min_pad = -1;
  for (int i = 0; i < 4; ++i) {
    if (cands[i] > max_bn) continue;
    const long pad = (long)((a->N + cands[i] - 1) / cands[i]) * cands[i];
    if (min_pad < 0 || pad < min_pad) min_pad = pad;
  }
  Plan best = {fixed_bn ? fixed_bn : 128, false};
  double best_cost = -1;
  for (int i = 0; i < 4; ++i) {
    const int bn = cands[i];
    if ((fixed_bn && bn != fixed_bn) || bn > max_bn) continue;
    if (!fixed_bn && a->N <= 128 && bn != 128) continue;
    const long pad = (long)((a->N + bn - 1) / bn) * bn;
    if (!fixed_bn && pad > min_pad + min_pad / 14) continue;  // more than ~7 % wasted columns
    const long T = (long)((a->N + bn - 1) / bn) * m_tiles;
    const double t_kb = fmax(2.0 * bn, (16384.0 + 128.0 * bn) / 80.0);
    const double t_epi = 1500.0 * bn / 32.0;
    const double t_tile = KB * t_kb + 600.0;
    const long rounds = (T + sms - 1) / sms;
    const double cost_dp = rounds * t_tile + t_epi;
    if (best_cost < 0 || cost_dp < best_cost) {
      best_cost = cost_dp;
      best = {bn, false};
    }
    if (KB >= 8 && (T % sms) != 0 && T * KB >= sms) {
      const long full = T / sms;
      const long t_dp = full >= 2 ? (full - 1) * sms : 0;
      const long t_sk = T - t_dp;
      const double followers = t_sk < sms ? (double)(sms - t_sk) / t_sk : 1.0;
      const double cost_sk = (full >= 2 ? (full - 1) : 0) * t_tile + (double)t_sk * KB / sms * t_kb + t_epi + 20000.0 +
                             followers * 128.0 * bn * 4.0 / 40.0;
      if (cost_sk < best_cost) {
        best_cost = cost_sk;
        best = {bn, true};
      }
    }
  }
  if (force) {
    int fbn = 0, fsk = 0;
    if (sscanf(force, "%d,%d", &fbn, &fsk) == 2) {
      if (!fixed_bn && fbn <= max_bn && (fbn == 256 || fbn == 192 || fbn == 160 || fbn == 128)) best.bn = fbn;
      best.sk = fsk != 0;
    }
  }
  return best;
}

struct Resolved {
  int bn, mode;
  bool sk;
};

static Resolved resolve(const idiff_gemm_args* a) {
  // GEGLU: one 256-column accumulator tile = 128 value columns + their 128 gates (packing.py)
  if (a->flags & IDIFF_EPI_GEGLU) return {256, MODE_GEGLU, plan_gemm(a, 256).sk};
  if (a->flags & IDIFF_OUT_F32_NCHW) return {128, MODE_NCHW, plan_gemm(a, 128).sk};
  // MODE_GATED stays at BN <= 192: its 256-wide instantiation spills (ptxas -v), the narrower ones do not
  if (a->gate_b) {
    const Plan pl = plan_gemm(a, 0, 192);
    return {pl.bn, MODE_GATED, pl.sk};
  }
  const Plan pl = plan_gemm(a, 0);
  return {pl.bn, MODE_PLAIN, pl.sk};
}

template <int MODE>
static int launch_bn(const idiff_gemm_args* a, cudaStream_t stream, const Resolved& r) {
  switch (r.bn) {
    case 256:
      if constexpr (MODE != MODE_GATED) return launch<256, MODE>(a, stream, r.sk);
      return -1;  // (resolve never plans it)
    case 192: return launch<192, MODE>(a, stream, r.sk);
    case 160: return launch<160, MODE>(a, stream, r.sk);
    default: return launch<128, MODE>(a, stream, r.sk);
  }
}

// One instantiation per (tile width, epilogue mode): each kernel carries only its own mode's code.
int gemm_v2(const idiff_gemm_args* a, cudaStream_t stream) {
  const Resolved r = resolve(a);
  if (r.mode == MODE_GEGLU) return launch<256, MODE_GEGLU>(a, stream, r.sk);
  if (r.mode == MODE_NCHW) return launch<128, MODE_NCHW>(a, stream, r.sk);
  if (r.mode == MODE_GATED) return launch_bn<MODE_GATED>(a, stream, r);
  return launch_bn<MODE_PLAIN>(a, stream, r);
}

// slots of the LayerNorm partial statistics a producer GEMM with these arguments writes per row
int ln_slots_of(const idiff_gemm_args* a) {
  const Resolved r = resolve(a);
  return (a->N + r.bn - 1) / r.bn;
}

}  // namespace v2
}  // namespace idiff

extern "C" int idiff_gemm(const idiff_gemm_args* a, void* stream) {
  using namespace idiff;
  IDIFF_REQUIRE(a && a->a && a->w && a->out, "idiff_gemm: null pointer argument");
  IDIFF_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0, "idiff_gemm: bad shape M=%d N=%d K=%d", a->M, a->N, a->K);
  const bool geglu = (a->flags & IDIFF_EPI_GEGLU) != 0;
  const bool nchw = (a->flags & IDIFF_OUT_F32_NCHW) != 0;
  if (geglu) {
    IDIFF_REQUIRE(a->N % 256 == 0, "idiff_gemm: GEGLU needs N %% 256 == 0 (N=%d)", a->N);
    IDIFF_REQUIRE(!a->residual && !a->rowadd && !nchw, "idiff_gemm: GEGLU excludes residual/rowadd/NCHW");
  }
  if (!nchw) {
    IDIFF_REQUIRE(a->N % 8 == 0, "idiff_gemm: N=%d must be a multiple of 8 for fp16 output", a->N);
    IDIFF_REQUIRE(a->ldo % 8 == 0, "idiff_gemm: ldo=%d must be a multiple of 8", a->ldo);
    IDIFF_REQUIRE((reinterpret_cast<uintptr_t>(a->out) & 15) == 0, "idiff_gemm: out not 16B aligned");
    if (a->residual) {
      IDIFF_REQUIRE(a->ldr % 8 == 0 && (reinterpret_cast<uintptr_t>(a->residual) & 15) == 0,
                    "idiff_gemm: residual must be 16B aligned with ldr %% 8 == 0");
    }
  } else {
    IDIFF_REQUIRE(!a->residual, "idiff_gemm: NCHW fp32 output excludes residual");
  }
  if (a->gate_b) {
    IDIFF_REQUIRE(a->residual, "idiff_gemm: gate_b scales the gated residual and needs a residual");
    IDIFF_REQUIRE(!a->rowadd && !a->ln_stats_in && !(a->flags & (IDIFF_EPI_SILU | IDIFF_EPI_GELU)),
                  "idiff_gemm: gate_b combines with bias, residual and ln_stats_out only");
  }
  if (a->workspace) {
    IDIFF_REQUIRE((reinterpret_cast<uintptr_t>(a->workspace) & 255) == 0, "idiff_gemm: workspace must be 256B aligned");
  }
  if (a->ln_stats_in) {
    IDIFF_REQUIRE(a->ln_colsum && a->ln_slots_in > 0 && a->ln_slots_in <= 64, "idiff_gemm: LayerNorm fold needs ln_colsum and 1..64 slots");
    IDIFF_REQUIRE(a->conv_h == 0 && !nchw && !a->rowadd, "idiff_gemm: LayerNorm fold applies to plain / GEGLU linear layers");
    IDIFF_REQUIRE((a->K + 63) / 64 <= 40, "idiff_gemm: LayerNorm fold needs K <= 2560 (K=%d)", a->K);
    IDIFF_REQUIRE((reinterpret_cast<uintptr_t>(a->ln_stats_in) & 7) == 0, "idiff_gemm: ln_stats_in must be 8B aligned");
  }
  if (a->ln_stats_out) {
    IDIFF_REQUIRE(a->conv_h == 0 && !nchw && !geglu, "idiff_gemm: row statistics are produced by plain linear layers");
    IDIFF_REQUIRE((reinterpret_cast<uintptr_t>(a->ln_stats_out) & 7) == 0, "idiff_gemm: ln_stats_out must be 8B aligned");
  }
  return v2::gemm_v2(a, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int idiff_gemm_ln_slots(const idiff_gemm_args* a) {
  using namespace idiff;
  IDIFF_REQUIRE(a && a->M > 0 && a->N > 0 && a->K > 0, "idiff_gemm_ln_slots: bad arguments");
  return v2::ln_slots_of(a);
}

extern "C" int idiff_set_gemm_workspace(void* ptr, long bytes) {
  using namespace idiff;
  if (ptr) {
    IDIFF_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 255) == 0, "idiff_set_gemm_workspace: pointer must be 256B aligned");
    // flags live inside the workspace and must start at zero
    IDIFF_CHECK_CUDA(cudaMemset(ptr, 0, (size_t)bytes));
  }
  v2::g_ws = ptr;
  v2::g_ws_bytes = ptr ? bytes : 0;
  return 0;
}

// Debug / profiling hook: when set, every GEMM CTA writes %globaltimer stamps to trace[cta*16 ..]: slot 0
// kernel entry, slot 7 exit, slots 12 / 13 the SM clock at entry / exit; for the CTA's first epilogue tile
// slots 1 / 2 / 3 = mainloop done / epilogue staged in shared memory / TMA store issued, slots 4 / 5 / 6 the
// same for its last one (a CTA without an epilogue tile leaves them 0).  NULL disables.
extern "C" int idiff_set_gemm_trace(void* ptr) {
  idiff::v2::g_trace = reinterpret_cast<unsigned long long*>(ptr);
  return 0;
}

extern "C" long idiff_gemm_workspace_bytes(void) {
  // up to 256 SMs x 128 x 256 fp32 partial tiles + flags
  return 256L * 128 * 256 * 4 + (1 << 20);
}
