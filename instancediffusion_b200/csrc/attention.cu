// Flash-style attention on wgmma for sm_90a: O = softmax(Q K^T * scale) V per (batch, head).
//
// One CTA owns a query tile of one (batch, head): warpgroup 0 is the TMA producer (Q once, then
// K / V tiles of 128 keys at d = 40, 64 keys otherwise, through a ring), and each consumer warpgroup
// owns 64 query rows: three of them (a 192-query tile) at d = 40, two (128 queries) otherwise.  Per key
// block a consumer warpgroup computes S = Q K^T with wgmma (Q and K from 128B-swizzled shared memory)
// into registers, runs the online softmax on the fragments (a row lives in the four threads of a quad),
// and feeds P straight from registers as the A operand of O += P V at N = d; V is consumed as an
// MN-major B operand from its token-major tile, so no transposed copy of V is ever made.  With two
// consumer warpgroups the PV product of block j - 1 runs on the tensor cores during the softmax of
// block j; with three, the other warpgroups' work fills that time.  O stays in registers and is
// normalised and stored at the end.
// Keys/values are read from up to two segments (visual tokens, then the 184 UniFusion object
// tokens of GatedSelfAttentionDense) -- the concatenation of attention.py:306 never exists.
// The optional instance-isolation mask (attention.py:187-255) is applied to the scores: query i may
// attend key j iff (mask_q[b][i] & mask_k[b][j]) != 0, or j is the visual token i itself.
//
// Replaces F.scaled_dot_product_attention at attention.py:134-144, 257-267 (+ the head
// split/merge permutes at :130-132,144,183-185,267).
#include "../../include/idiff_b200.h"
#include "common.cuh"
#include "host.cuh"
#include "wgmma.cuh"

namespace idiff {

struct AttnKParams {
  int heads, nq, n0, n1, kv1_broadcast;
  float scale_log2e;
  h16* out;
  int out_ld;
  const uint32_t* mask_q;  // [batch][nq] or null
  const uint32_t* mask_k;  // [batch][n0 + n1]
};

template <int D>
struct AttnCfg {
  static constexpr int ND = (D + 63) / 64;           // 64-wide d chunks (one TMA box each)
  static constexpr int KSTEPS = (D + 15) / 16;       // wgmma k-steps of QK^T (zero padded)
  // keys per block: at d = 40 a 64-key block is too little work to amortise a block's fixed cost (ring
  // waits, wgmma issue and latency, row-max shuffles, O rescale); at d >= 80 S + P + O must fit in registers
  static constexpr int BKV = (D <= 64) ? 128 : 64;
  static constexpr int STAGES = (D <= 64) ? 4 : 3;
  // consumer warpgroups of 64 query rows.  At d = 40 a row's softmax is a long dependent chain (max, subtract,
  // exp2, row sum, pack) next to little tensor work, so a third warpgroup gives each scheduler another
  // independent softmax warp to issue from; at d >= 80 the S + P + O fragments need 232 registers a thread.
  static constexpr int NCW = (D <= 64) ? 3 : 2;
  static constexpr int BQ = 64 * NCW;
  static constexpr int THREADS = 128 * (NCW + 1);
  // register split (setmaxnreg at the head of each role branch): 128 x PRODUCER + 128 NCW x CONSUMER <= 65536
  static constexpr int PRODUCER_REGS = (NCW == 3) ? 24 : 40;
  static constexpr int CONSUMER_REGS = (NCW == 3) ? 160 : 232;
  static_assert(128 * PRODUCER_REGS + 128 * NCW * CONSUMER_REGS <= 65536, "register split");
  // With two consumer warpgroups each one also keeps its own PV product of block j - 1 on the tensor cores while
  // it runs the softmax of block j, which keeps P_{j-1} (BKV / 4 registers) live next to S_j.  ptxas allocates
  // no thread more than the launch bound's 65536 / THREADS registers whatever setmaxnreg grants (128 at 512
  // threads), and that loop needs about 140 at d = 40; with three warpgroups a consumer waits for its PV
  // product before the softmax, and the other two warpgroups' wgmmas and softmaxes fill the wait.
  static constexpr bool PV_UNDER_SOFTMAX = NCW == 2;
  static constexpr int Q_BYTES = ND * BQ * 128;
  static constexpr int KV_TILE_BYTES = ND * BKV * 128;  // one of K or V
  static constexpr int SMEM_BYTES = 1024 + Q_BYTES + STAGES * 2 * KV_TILE_BYTES + 256;  // + alignment slack, barriers
};

// P is stored as 2^(s*c - m*c + P_LOG2_BIAS) <= 2^15 before it is rounded to 16 bits: unbiased, fp16 P would go
// subnormal (an absolute step of 2^-24) for keys more than 2^-14 below the row max, and the sum of those rounding errors
// over thousands of keys can exceed the relative precision of the output.  With the bias fp16 P stays normal down to
// 2^-29 of the max.  The bias scales O and l alike and cancels in O / l; alpha is a difference of maxima and unaffected.
constexpr float P_LOG2_BIAS = 15.f;

template <int D, bool MASKED>
__global__ void __launch_bounds__(AttnCfg<D>::THREADS, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK0,
                 const __grid_constant__ CUtensorMap tmV0, const __grid_constant__ CUtensorMap tmK1,
                 const __grid_constant__ CUtensorMap tmV1, const AttnKParams p) {
  using Cfg = AttnCfg<D>;
  constexpr int ND = Cfg::ND, STAGES = Cfg::STAGES, BKV = Cfg::BKV, NCW = Cfg::NCW, BQ = Cfg::BQ;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Cfg::Q_BYTES;
  uint8_t* sV = sK + STAGES * Cfg::KV_TILE_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + STAGES * Cfg::KV_TILE_BYTES);
  uint64_t* q_full = bars;                 // 1
  uint64_t* k_full = bars + 1;             // STAGES
  uint64_t* v_full = k_full + STAGES;      // STAGES
  uint64_t* kv_empty = v_full + STAGES;    // STAGES (one arrival per consumer warp)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * BQ;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int T0 = (p.n0 + BKV - 1) / BKV;
  const int T1 = (p.n1 + BKV - 1) / BKV;
  const int T = T0 + T1;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK0);
    tma_prefetch_desc(&tmV0);
    mbar_init(q_full, 1);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&v_full[s], 1);
      mbar_init(&kv_empty[s], 4 * NCW);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(Cfg::PRODUCER_REGS));
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      mbar_expect_tx(q_full, Cfg::Q_BYTES);
      for (int c = 0; c < ND; ++c) tma_load_4d(sQ + c * BQ * 128, &tmQ, q_full, c * 64, h, q0, b);
      uint32_t s = 0, ph = 0;
      for (int j = 0; j < T; ++j) {
        mbar_wait(&kv_empty[s], ph ^ 1);
        const bool seg1 = j >= T0;
        const int row = (seg1 ? (j - T0) : j) * BKV;
        const int bb = seg1 ? (p.kv1_broadcast ? 0 : b) : b;
        const CUtensorMap* mk = seg1 ? &tmK1 : &tmK0;
        const CUtensorMap* mv = seg1 ? &tmV1 : &tmV0;
        mbar_expect_tx(&k_full[s], Cfg::KV_TILE_BYTES);
        for (int c = 0; c < ND; ++c)
          tma_load_4d(sK + s * Cfg::KV_TILE_BYTES + c * BKV * 128, mk, &k_full[s], c * 64, h, row, bb);
        mbar_expect_tx(&v_full[s], Cfg::KV_TILE_BYTES);
        for (int c = 0; c < ND; ++c)
          tma_load_4d(sV + s * Cfg::KV_TILE_BYTES + c * BKV * 128, mv, &v_full[s], c * 64, h, row, bb);
        if (++s == STAGES) {
          s = 0;
          ph ^= 1;
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(Cfg::CONSUMER_REGS));
    // ===================== consumers: S = Q K^T, online softmax, O += P V =====================
    // Per key block j a consumer issues S_j = Q K_j^T and O += P_{j-1} V_{j-1} back to back, runs the
    // softmax of S_j while the PV product is still on the tensor cores, then waits for it and rescales O
    // (PV_UNDER_SOFTMAX; otherwise PV_{j-1} retires before S_j is issued, and O is rescaled after the softmax).
    // The consumer warpgroups also take turns issuing, round robin (named barrier 1 + cw grants warpgroup cw
    // its turn; each turn grants the next warpgroup's), so one warpgroup's softmax runs under the others' wgmmas.
    const int cw = (warp >> 2) - 1;  // rows [64 cw, 64 cw + 64) of the query tile
    const uint32_t my_turn = 1 + cw, next_turn = 1 + (cw + 1) % NCW;
    if (cw == NCW - 1) named_bar_arrive(1, 256);  // warpgroup 0 takes the first turn
    if (q0 + cw * 64 >= p.nq) {
      // every row of this warpgroup lies past nq (the last tile of a ragged nq): no math, but it still takes
      // its T + 1 turns and releases each K/V stage once that stage's fill has landed, as the loop below does
      uint32_t s = 0, ph = 0;
      for (int j = 0; j <= T; ++j) {
        named_bar_sync(my_turn, 256);
        if (j < T || cw != NCW - 1) named_bar_arrive(next_turn, 256);
        if (j < T) {
          mbar_wait(&v_full[s], ph);
          if (lane == 0) mbar_arrive(&kv_empty[s]);
          if (++s == STAGES) {
            s = 0;
            ph ^= 1;
          }
        }
      }
      return;
    }
    const int t4 = lane & 3;
    const int rl0 = cw * 64 + (warp & 3) * 16 + (lane >> 2);  // tile rows of this thread: rl0, rl0 + 8
    const float c = p.scale_log2e;
    // descriptors: Q / K K-major (rows of 128 B, 8-row atoms 1024 B apart); V MN-major (64-wide d atoms
    // BKV * 128 B apart, 8-key groups 1024 B apart).  The PV product runs at N = D: it reads the first D
    // columns of the zero-padded 64-wide V boxes.
    const uint64_t dq = make_wgmma_desc(smem_u32(sQ) + cw * 64 * 128, 16, 1024);
    const uint64_t dk = make_wgmma_desc(smem_u32(sK), 16, 1024);
    const uint64_t dv = make_wgmma_desc(smem_u32(sV), BKV * 128, 1024);

    uint32_t qword[2] = {0xffffffffu, 0xffffffffu};
    if (MASKED) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int qr = q0 + rl0 + 8 * hh;
        qword[hh] = qr < p.nq ? __ldg(p.mask_q + (long)b * p.nq + qr) : 0xffffffffu;
      }
    }
    float o[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY};
    float l_part[2] = {0.f, 0.f};  // this thread's share of the row sums (quad-reduced at the end)
    float sc[BKV / 2];
    float alpha[2];

    auto issue_qk = [&](uint32_t st) {
#pragma unroll
      for (int kk = 0; kk < Cfg::KSTEPS; ++kk)
        Wgmma<BKV>::ss(sc, dq + (((kk >> 2) * BQ * 128 + (kk & 3) * 32) >> 4),
                       dk + ((st * Cfg::KV_TILE_BYTES + (kk >> 2) * BKV * 128 + (kk & 3) * 32) >> 4), kk > 0 ? 1u : 0u);
      wgmma_commit();
    };
    auto issue_pv = [&](const uint32_t (&pa)[BKV / 16][4], uint32_t st) {
#pragma unroll
      for (int kk = 0; kk < BKV / 16; ++kk)
        Wgmma<D>::rs(o, pa[kk], dv + ((st * Cfg::KV_TILE_BYTES + kk * 16 * 128) >> 4), 1u);
      wgmma_commit();
    };
    // online softmax of the scores of key block j (rows rl0, rl0 + 8; a row's BKV scores are spread over
    // the quad): sc becomes P = 2^(s*c - m*c + P_LOG2_BIAS) in place, alpha the factor O has to be rescaled by
    auto softmax = [&](int j) {
      const bool seg1 = j >= T0;
      const int key0 = seg1 ? (j - T0) * BKV : j * BKV;  // first key of the block within its segment
      const int nv = min(BKV, (seg1 ? p.n1 : p.n0) - key0);
      // (MASKED) keys this row may not see, and keys past the segment end (its last block only), score -inf
      if (MASKED) {
#pragma unroll
        for (int jj = 0; jj < BKV / 8; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int kc = 8 * jj + 2 * t4 + e;  // key column of the block
            if (kc < nv) {
              const uint32_t kw = __ldg(p.mask_k + (long)b * (p.n0 + p.n1) + (seg1 ? p.n0 : 0) + key0 + kc);
#pragma unroll
              for (int hh = 0; hh < 2; ++hh) {
                const bool self = !seg1 && key0 + kc == q0 + rl0 + 8 * hh;
                if ((kw & qword[hh]) == 0u && !self) sc[4 * jj + 2 * hh + e] = -INFINITY;
              }
            }
          }
        }
      }
      if (nv < BKV) {
#pragma unroll
        for (int jj = 0; jj < BKV / 8; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (8 * jj + 2 * t4 + e >= nv) {
              sc[4 * jj + e] = -INFINITY;
              sc[4 * jj + 2 + e] = -INFINITY;
            }
          }
        }
      }
      float mc[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        // pairwise tree (a max is exact in any order): a log-depth dependency chain instead of a serial one
        float m8[BKV / 8];
#pragma unroll
        for (int jj = 0; jj < BKV / 8; ++jj) m8[jj] = fmaxf(sc[4 * jj + 2 * hh], sc[4 * jj + 2 * hh + 1]);
        static_assert(BKV == 64 || BKV == 128, "row-max tree depth");
#pragma unroll
        for (int jj = 0; jj < BKV / 16; ++jj) m8[jj] = fmaxf(m8[jj], m8[jj + BKV / 16]);
#pragma unroll
        for (int jj = 0; jj < BKV / 32; ++jj) m8[jj] = fmaxf(m8[jj], m8[jj + BKV / 32]);
#pragma unroll
        for (int jj = 0; jj < BKV / 64; ++jj) m8[jj] = fmaxf(m8[jj], m8[jj + BKV / 64]);
        if (BKV == 128) m8[0] = fmaxf(m8[0], m8[1]);
        float mx = m8[0];
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m_run[hh], mx);
        // a row that has seen no live key yet keeps 0 as its reference: P = 0 instead of NaN
        const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
        alpha[hh] = exp2_approx((m_run[hh] - m_use) * c);  // m_run = -inf -> 0
        m_run[hh] = m_new;
        mc[hh] = fmaf(m_use, c, -P_LOG2_BIAS);
        l_part[hh] *= alpha[hh];
      }
#pragma unroll
      for (int jj = 0; jj < BKV / 8; ++jj) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          float& p0 = sc[4 * jj + 2 * hh];
          float& p1 = sc[4 * jj + 2 * hh + 1];
          p0 = exp2_approx(fmaf(p0, c, -mc[hh]));
          p1 = exp2_approx(fmaf(p1, c, -mc[hh]));
          l_part[hh] += p0 + p1;
        }
      }
    };
    // P as the 16-bit A fragments of the BKV / 16 k-steps of 16 keys: register r of k-step kk = accumulator group
    // 2kk + (r >> 1), row half (r & 1).  Written only once the previous PV product (which reads pa) retired.
    uint32_t pa[BKV / 16][4];
    auto pack_p = [&]() {
#pragma unroll
      for (int kk = 0; kk < BKV / 16; ++kk)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int jj = 2 * kk + (r >> 1), hh = r & 1;
          pa[kk][r] = pack_half2(sc[4 * jj + 2 * hh], sc[4 * jj + 2 * hh + 1]);
        }
    };

    // rescale O by the factor of the block just through the softmax and pack its P
    auto rescale_pack = [&]() {
      // alpha is exactly 1 where the row max did not move (most blocks once a row has seen a few):
      // skip the multiply when that holds for every row of the warp
      if (!__all_sync(0xffffffffu, alpha[0] == 1.f && alpha[1] == 1.f)) {
#pragma unroll
        for (int jj = 0; jj < D / 8; ++jj) {
          o[4 * jj] *= alpha[0];
          o[4 * jj + 1] *= alpha[0];
          o[4 * jj + 2] *= alpha[1];
          o[4 * jj + 3] *= alpha[1];
        }
      }
      pack_p();
    };
    // PV_{j-2} has retired: free its K/V stage, rescale O by the factor of block j - 1 and pack P_{j-1}.
    // Called at the top of a trip, not after the softmax: the compiler must not hoist the wait into the
    // softmax (where it would stall on the PV product the softmax is meant to hide).
    auto retire_pv = [&](bool release, uint32_t st) {
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      if (release && lane == 0) mbar_arrive(&kv_empty[st]);
      rescale_pack();
    };

    mbar_wait(q_full, 0);
    named_bar_sync(my_turn, 256);
    mbar_wait(&k_full[0], 0);
    wgmma_fence();
    issue_qk(0);
    named_bar_arrive(next_turn, 256);
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    softmax(0);
    if (!Cfg::PV_UNDER_SOFTMAX) rescale_pack();
    uint32_t s = 0, ph = 0;  // ring stage / phase of block j - 1
    uint32_t s_prev = 0;     // ring stage of block j - 2
    for (int j = 1; j < T; ++j) {
      if (Cfg::PV_UNDER_SOFTMAX) retire_pv(j >= 2, s_prev);
      const uint32_t sn = (s + 1 == STAGES) ? 0u : s + 1, phn = (sn == 0) ? ph ^ 1u : ph;
      named_bar_sync(my_turn, 256);
      if (Cfg::PV_UNDER_SOFTMAX) {
        mbar_wait(&k_full[sn], phn);
        wgmma_fence();
        issue_qk(sn);
        mbar_wait(&v_full[s], ph);
        wgmma_fence();  // ptxas would otherwise insert this fence itself after the wait loop
        issue_pv(pa, s);
        named_bar_arrive(next_turn, 256);
        wgmma_wait<1>();  // S_j has landed; PV_{j-1} may still run
        wgmma_fence_regs(sc);
        softmax(j);
      } else {
        // PV_{j-1} retires before S_j is issued: P_{j-1} and S_j never hold registers at the same time
        mbar_wait(&v_full[s], ph);
        wgmma_fence();
        issue_pv(pa, s);
        wgmma_wait<0>();
        wgmma_fence_regs(o);
        if (lane == 0) mbar_arrive(&kv_empty[s]);
        mbar_wait(&k_full[sn], phn);
        wgmma_fence();
        issue_qk(sn);
        named_bar_arrive(next_turn, 256);
        wgmma_wait<0>();
        wgmma_fence_regs(sc);
        softmax(j);
        rescale_pack();
      }
      s_prev = s;
      s = sn;
      ph = phn;
    }
    if (Cfg::PV_UNDER_SOFTMAX) retire_pv(T >= 2, s_prev);
    // the last PV product; the last warpgroup's turn is the last of all, so it grants none
    named_bar_sync(my_turn, 256);
    mbar_wait(&v_full[s], ph);
    wgmma_fence();
    issue_pv(pa, s);
    if (cw != NCW - 1) named_bar_arrive(next_turn, 256);
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    if (lane == 0) mbar_arrive(&kv_empty[s]);

    // epilogue: O / l -> 16-bit
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float l = l_part[hh];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const float inv_l = 1.0f / l;
      const int qrow = q0 + rl0 + 8 * hh;
      if (qrow >= p.nq) continue;
      h16* orow = p.out + ((long)b * p.nq + qrow) * p.out_ld + h * D;
#pragma unroll
      for (int jj = 0; jj < D / 8; ++jj)
        *reinterpret_cast<uint32_t*>(orow + 8 * jj + 2 * t4) =
            pack_half2(o[4 * jj + 2 * hh] * inv_l, o[4 * jj + 2 * hh + 1] * inv_l);
    }
  }
}

// 4-D view (d, head, token, batch) of an fp16 [batch*rows, ld] matrix whose head h occupies
// columns [h*d, (h+1)*d) from `base`.
static int make_head_tmap(CUtensorMap* m, const void* base, int d, int heads, int rows, int batch,
                          int ld, int box_rows) {
  const uint64_t dims[4] = {(uint64_t)d, (uint64_t)heads, (uint64_t)rows, (uint64_t)batch};
  const uint64_t strides[3] = {(uint64_t)d * 2, (uint64_t)ld * 2, (uint64_t)rows * ld * 2};
  const uint32_t box[4] = {64u, 1u, (uint32_t)box_rows, 1u};
  return encode_tmap_f16(m, base, 4, dims, strides, box);
}

template <int D, bool MASKED>
static int launch_attention(const idiff_attn_args* a, cudaStream_t stream) {
  using Cfg = AttnCfg<D>;
  CUtensorMap tmQ, tmK0, tmV0, tmK1, tmV1;
  if (make_head_tmap(&tmQ, a->q, D, a->heads, a->nq, a->batch, a->q_ld, Cfg::BQ)) return -1;
  if (make_head_tmap(&tmK0, a->k0, D, a->heads, a->n0, a->batch, a->k0_ld, Cfg::BKV)) return -1;
  if (make_head_tmap(&tmV0, a->v0, D, a->heads, a->n0, a->batch, a->v0_ld, Cfg::BKV)) return -1;
  if (a->n1 > 0) {
    const int b1 = a->kv1_batch == 1 ? 1 : a->batch;
    if (make_head_tmap(&tmK1, a->k1, D, a->heads, a->n1, b1, a->k1_ld, Cfg::BKV)) return -1;
    if (make_head_tmap(&tmV1, a->v1, D, a->heads, a->n1, b1, a->v1_ld, Cfg::BKV)) return -1;
  } else {
    tmK1 = tmK0;
    tmV1 = tmV0;
  }
  AttnKParams p;
  p.heads = a->heads;
  p.nq = a->nq;
  p.n0 = a->n0;
  p.n1 = a->n1;
  p.kv1_broadcast = (a->kv1_batch == 1) ? 1 : 0;
  p.scale_log2e = a->scale * 1.4426950408889634f;
  p.out = reinterpret_cast<h16*>(a->out);
  p.out_ld = a->out_ld;
  p.mask_q = reinterpret_cast<const uint32_t*>(a->mask_q);
  p.mask_k = reinterpret_cast<const uint32_t*>(a->mask_k);
  static bool attr_set = false;
  if (!attr_set) {
    IDIFF_CHECK_CUDA(cudaFuncSetAttribute(attention_kernel<D, MASKED>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          Cfg::SMEM_BYTES));
    attr_set = true;
  }
  dim3 grid((a->nq + Cfg::BQ - 1) / Cfg::BQ, a->heads, a->batch);
  IDIFF_CHECK_CUDA(launch(attention_kernel<D, MASKED>, dim3(grid), dim3(Cfg::THREADS), Cfg::SMEM_BYTES, stream, tmQ,
                          tmK0, tmV0, tmK1, tmV1, p));
  return 0;
}

}  // namespace idiff

extern "C" int idiff_attention(const idiff_attn_args* a, void* stream) {
  using namespace idiff;
  IDIFF_REQUIRE(a && a->q && a->k0 && a->v0 && a->out, "idiff_attention: null pointer argument");
  IDIFF_REQUIRE(a->nq > 0 && a->n0 > 0 && a->n1 >= 0 && a->batch > 0 && a->heads > 0,
                "idiff_attention: bad shape");
  IDIFF_REQUIRE(a->n1 == 0 || (a->k1 && a->v1), "idiff_attention: segment 1 pointers missing");
  IDIFF_REQUIRE(a->out_ld % 8 == 0 && (reinterpret_cast<uintptr_t>(a->out) & 15) == 0,
                "idiff_attention: out must be 16B aligned, out_ld %% 8 == 0");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (a->mask_q || a->mask_k) {
    IDIFF_REQUIRE(a->mask_q && a->mask_k, "idiff_attention: mask_q and mask_k come together");
    IDIFF_REQUIRE(a->head_dim == 40, "idiff_attention: the instance-isolation mask exists at the 64x64 level only "
                                     "(head_dim 40; attention.py:197), got head_dim %d", a->head_dim);
    IDIFF_REQUIRE(a->n0 % 4 == 0 && (a->n0 + a->n1) % 4 == 0 && (reinterpret_cast<uintptr_t>(a->mask_k) & 15) == 0,
                  "idiff_attention: mask_k must be 16B aligned with n0 and n0 + n1 multiples of 4");
    return launch_attention<40, true>(a, s);
  }
  switch (a->head_dim) {
    case 40: return launch_attention<40, false>(a, s);
    case 80: return launch_attention<80, false>(a, s);
    case 160: return launch_attention<160, false>(a, s);
    default: return set_error("idiff_attention: unsupported head_dim %d (40/80/160)", a->head_dim);
  }
}
