// CRF Viterbi decode for sm_90a — replaces tf.contrib.crf.crf_decode as called at
// reference tools/layer.py:140-142 (semantics restated in SURVEY.md Appendix A.1).
//
// viterbi_plan() below picks the kernel from (B, L, K, alignment of logits, number of SMs) alone; the first row whose
// condition holds wins.  big = B > 64 * num_sms; every kernel also needs its shared memory to fit in 227 KB.
//
//   plan         kernel                       picked when                       backpointers live in           shared memory per CTA
//   SMALL        crf_viterbi_lanes_kernel     B <= 4096                         smem, 1 byte per lane          (32 + 4 SPW) L
//                (crf_small.cu, lane per tag)
//   TMA          crf_viterbi_tma_kernel       big, K <= 16, L*K % 4 == 0,       smem, 4 bits per tag           (160 + 32 HB) L + 0.3 KB
//                <K, 32, 2, 2, 8>             logits 16-byte aligned                                           (L <= 1208 at K = 10)
//   PARKED       crf_viterbi_gs_kernel        big, K <= 16, TMA ruled out       tags 0..7: the CTA's slab of   64 (1 + HB) L + 1 KB
//                <K, 64, 4, 6>                (L*K % 4, alignment, L)           tags_out; tags 8..15: smem     (L <= 1808 at K = 10)
//   ONCHIP_128   crf_viterbi_kernel<K, 128>   big (K > 16, or PARKED too long)  smem, 4 or 8 bits per tag      516 W L + ring (4 KB * (2K|1))
//   ONCHIP_32    crf_viterbi_kernel<K, 32>    any B                             the same                       132 W L + ring / 4
//   SMALL_ANY_B  crf_viterbi_lanes_kernel     B > 4096, L past all the above    as SMALL                       as SMALL
//
// (SPW = Lanes<K>::SPW sequences per warp, HB = BpSplit<K>::HB bytes of high nibbles per step, W = BpPack<K>::W words
// per step.)  Every kernel but the lane-per-tag one walks one sequence per thread with the K-wide max-plus state in
// registers.  PARKED exists because the all-on-chip kernel, which would otherwise serve its calls, is slower on them:
// on an H100 SXM (80 GB HBM3, 700 W limit), ragged lengths, (B, L, K) = (19000, 150, 7): 0.228 ms against 0.158 ms
// (1.45x); (262144, 127, 10): 2.22 ms against 1.25 ms (1.78x); (9490, 9, 3): 1.17x; only at (9600, 37, 7) is it 4.5 %
// faster (scripts/bench_crf_dispatch.py).
//
// Bit-exactness contract (tests/test_crf_gpu.py): fp32 adds in the reference order
// (s[i] + trans[i][j], max over i, then + logits[t][j]); ties -> lowest index (strict >).
#include <type_traits>

#include "crf_common.cuh"
#include "tc_common.cuh"

namespace {

using namespace crf;

// ---------------------------------------------------------------------------------------------
// All-on-chip kernel: transition matrix in registers (K <= 10) or broadcast smem reads.  Backpointers never leave the
// SM: they are packed 4 bits (K <= 16) or 8 bits per tag into smem words laid out [t][w][thread], and the decoded tags
// are written back over word 0 of the same slots during the backtrace, so the final [NT, L] int32 store to HBM is fully
// coalesced.
template <int K>
struct BpPack {
  static constexpr int NIB = (K <= 16) ? 4 : 8;
  static constexpr int PER = 32 / NIB;
  static constexpr int W = (K + PER - 1) / PER;
  static constexpr uint32_t MASK = (1u << NIB) - 1u;
};

template <int K, int NT>
size_t viterbi_smem_bytes(int L) {
  using Gm = Geom<K>;
  size_t words = Gm::KK4 + NT + (size_t)NSTAGE * NT * Gm::P + (size_t)L * BpPack<K>::W * (NT + 1);
  return words * 4;
}

template <int K, int NT>
__global__ void __launch_bounds__(NT)
crf_viterbi_kernel(const float* __restrict__ logits, const int32_t* __restrict__ seq_len,
                   const float* __restrict__ trans, int32_t* __restrict__ tags_out,
                   float* __restrict__ best_score, int B, int L, int vec16) {
  using Gm = Geom<K>;
  using Bp = BpPack<K>;
  constexpr int T = Gm::T, G = Gm::G, P = Gm::P, W = Bp::W, NTP = NT + 1;
  constexpr bool TR_REGS = (K <= 10);
  constexpr int UNR = Gm::UNROLL ? K : 1;

  extern __shared__ __align__(16) float smem[];
  float* s_trT = smem;                                        // [j][i]
  int* s_len = reinterpret_cast<int*>(s_trT + Gm::KK4);       // [NT]
  float* s_stage = reinterpret_cast<float*>(s_len + NT);      // [NSTAGE][NT][P]
  uint32_t* s_bp = reinterpret_cast<uint32_t*>(s_stage + NSTAGE * NT * P);  // [L][W][NTP]

  const int tid = threadIdx.x;
  const int row0 = blockIdx.x * NT;
  const int nv = min(NT, B - row0);
  const int LK = L * K;

  for (int e = tid; e < K * K; e += NT) {
    const int i = e / K, j = e - i * K;
    s_trT[j * K + i] = trans[e];
  }
  int mylen = 1;
  if (tid < nv) mylen = clamp_len(seq_len, row0 + tid, L);
  s_len[tid] = mylen;
  const int bmax = block_max_int<NT>(tid < nv ? mylen : 1, reinterpret_cast<int*>(s_bp));
  // (block_max_int ends with __syncthreads: s_len / s_trT are visible)

  const float* gbase = logits + (size_t)row0 * LK;
  const int nchunk = (bmax + T - 1) / T;

#pragma unroll
  for (int s = 0; s < NSTAGE - 1; ++s) {
    if (s < nchunk) stage_logits<K, NT>(s_stage + s * NT * P, gbase, LK, s * T, L, nv, s_len, vec16);
    cp_async_commit();
  }

  float tr[TR_REGS ? K * K : 1];
  if (TR_REGS) {
#pragma unroll
    for (int e = 0; e < K * K; ++e) tr[e] = s_trT[e];
  }

  float s[K];
#pragma unroll UNR
  for (int j = 0; j < K; ++j) s[j] = 0.f;

  for (int c = 0; c < nchunk; ++c) {
    const int cn = c + NSTAGE - 1;
    if (cn < nchunk)
      stage_logits<K, NT>(s_stage + (cn % NSTAGE) * NT * P, gbase, LK, cn * T, L, nv, s_len, vec16);
    cp_async_commit();
    cp_async_wait<NSTAGE - 1>();
    __syncthreads();

    const int t0 = c * T;
    if (tid < nv && t0 < mylen) {
      const float* rowp = s_stage + (c % NSTAGE) * NT * P + tid * P;
#pragma unroll 1
      for (int g = 0; g < T / G; ++g) {
        if (t0 + g * G >= mylen) break;
        float xs[G * K];
        load_group<K>(xs, rowp, g);
#pragma unroll
        for (int gg = 0; gg < G; ++gg) {
          const int t = t0 + g * G + gg;
          if (t < mylen) {
            if (t == 0) {
#pragma unroll UNR
              for (int j = 0; j < K; ++j) s[j] = xs[gg * K + j];
            } else {
              // i-outer order: K independent (best, arg) pairs -> K-way ILP; per (i,j) the fp32 ops and the
              // strict '>' (first max wins) are exactly those of the reference recursion
              float best[K];
              int arg[K];
              uint32_t bpw[W];
#pragma unroll
              for (int w = 0; w < W; ++w) bpw[w] = 0u;
#pragma unroll UNR
              for (int j = 0; j < K; ++j) {
                best[j] = s[0] + (TR_REGS ? tr[j * K] : s_trT[j * K]);
                arg[j] = 0;
              }
#pragma unroll UNR
              for (int i = 1; i < K; ++i) {
#pragma unroll UNR
                for (int j = 0; j < K; ++j) {
                  const float v = s[i] + (TR_REGS ? tr[j * K + i] : s_trT[j * K + i]);
                  if (v > best[j]) {
                    best[j] = v;
                    arg[j] = i;
                  }
                }
              }
#pragma unroll UNR
              for (int j = 0; j < K; ++j) {
                s[j] = xs[gg * K + j] + best[j];
                bpw[j / Bp::PER] |= (uint32_t)arg[j] << ((j % Bp::PER) * Bp::NIB);
              }
#pragma unroll
              for (int w = 0; w < W; ++w) s_bp[(t * W + w) * NTP + tid] = bpw[w];
            }
          }
        }
      }
    }
    __syncthreads();
  }

  if (tid < nv) {
    float best;
    int y = argmax_first<K>(s, best);
    if (best_score != nullptr) best_score[row0 + tid] = best;
    for (int t = mylen - 1; t >= 1; --t) {
      const uint32_t w = s_bp[(t * W + y / Bp::PER) * NTP + tid];
      const int prev = (int)((w >> ((y % Bp::PER) * Bp::NIB)) & Bp::MASK);
      s_bp[(t * W) * NTP + tid] = (uint32_t)y;
      y = prev;
    }
    s_bp[tid] = (uint32_t)y;
  }
  __syncthreads();

  store_tags_coalesced<NT>(tags_out + (size_t)row0 * L, nv, L, s_len,
                           [&](int r, int p) { return (int)s_bp[(p * W) * NTP + r]; });
}

// ---------------------------------------------------------------------------------------------
// Occupancy-first variant (K <= 16): the 4-bit backpointers of tags 0..7 (one 32-bit word per
// step) are parked in the CTA's own [nv, L] slab of tags_out — exactly 4 bytes per step per
// sequence, written and read back by the same thread (coalesced [t][thread] layout, L2-resident
// for the CTA's lifetime) — and only the nibbles of tags 8..K-1 stay in shared memory.  Shared
// memory per CTA drops from ~219 KB to ~40 KB, so several CTAs share an SM and the per-step
// dependency chain of one warp is hidden behind the others (the all-on-chip kernel ran one warp
// per scheduler at IPC 1.5).  The s[i]+trans[i][j] adds are issued as FADD2 pairs; values, the
// strict '>' tie rule and the add order are unchanged (bit-exact contract above).
template <int K>
struct BpSplit {
  static constexpr int HB = (K <= 8) ? 0 : (K <= 10 ? 1 : (K <= 12 ? 2 : 4));  // on-chip bytes per step
};

template <int K, int NT, int TT>
size_t viterbi_gs_smem_bytes(int L) {
  using Gm = Geom<K, TT>;
  const size_t stage = (size_t)NSTAGE * NT * Gm::P * 4;
  const size_t dec = (size_t)NT * (((L + 3) & ~3) + 4);
  const size_t hi = ((size_t)L * NT * BpSplit<K>::HB + 15) & ~(size_t)15;
  return (size_t)(((2 * K * ((K + 1) / 2) + 3) & ~3) + NT) * 4 + (stage > dec ? stage : dec) + hi;
}

template <int K, int NT, int TT, int MINB>
__global__ void __launch_bounds__(NT, MINB)
crf_viterbi_gs_kernel(const float* __restrict__ logits, const int32_t* __restrict__ seq_len,
                      const float* __restrict__ trans, int32_t* tags_out,
                      float* __restrict__ best_score, int B, int L, int vec16) {
  using Gm = Geom<K, TT>;
  constexpr int T = Gm::T, G = Gm::G, P = Gm::P, KP = (K + 1) / 2, HB = BpSplit<K>::HB;
  constexpr bool TR_REGS = (K <= 10);
  constexpr int UNR = Gm::UNROLL ? K : 1;

  extern __shared__ __align__(16) float smem[];
  float* s_tr = smem;                                           // [i][2*KP]: trans rows, pad column = 0
  int* s_len = reinterpret_cast<int*>(s_tr + ((2 * K * KP + 3) & ~3));   // [NT]  (offset rounded: the ring below takes 16-byte cp.async / LDS.128)
  float* s_stage = reinterpret_cast<float*>(s_len + NT);        // [NSTAGE][NT][P]; reused as s_dec
  const int Lp = ((L + 3) & ~3) + 4;                            // byte pitch of a decoded row (Lp/4 odd-ish)
  const size_t stage_b = (size_t)NSTAGE * NT * P * 4, dec_b = (size_t)NT * Lp;
  uint8_t* s_dec = reinterpret_cast<uint8_t*>(s_stage);         // [NT][Lp] decoded tags (after the forward loop)
  uint8_t* s_hi = reinterpret_cast<uint8_t*>(s_stage) + (stage_b > dec_b ? stage_b : dec_b);  // [L][NT] x HB bytes

  const int tid = threadIdx.x;
  const int row0 = blockIdx.x * NT;
  const int nv = min(NT, B - row0);
  const int LK = L * K;

  for (int e = tid; e < K * 2 * KP; e += NT) {
    const int i = e / (2 * KP), j = e - i * 2 * KP;
    s_tr[e] = (j < K) ? trans[i * K + j] : 0.f;
  }
  int mylen = 1;
  if (tid < nv) mylen = clamp_len(seq_len, row0 + tid, L);
  s_len[tid] = mylen;
  const int bmax = block_max_int<NT>(tid < nv ? mylen : 1, reinterpret_cast<int*>(s_stage));

  const float* gbase = logits + (size_t)row0 * LK;
  uint32_t* scratch = reinterpret_cast<uint32_t*>(tags_out + (size_t)row0 * L);  // [L][nv] words of this CTA
  const int nchunk = (bmax + T - 1) / T;

#pragma unroll
  for (int s = 0; s < NSTAGE - 1; ++s) {
    if (s < nchunk) stage_logits<K, NT, TT>(s_stage + s * NT * P, gbase, LK, s * T, L, nv, s_len, vec16);
    cp_async_commit();
  }

  f32x2 tr2[TR_REGS ? K * KP : 1];
  if (TR_REGS) {
#pragma unroll
    for (int e = 0; e < K * KP; ++e) tr2[e] = pk2(s_tr[2 * e], s_tr[2 * e + 1]);
  }
  auto trp = [&](int i, int q) -> f32x2 {
    if (TR_REGS) return tr2[i * KP + q];
    return pk2(s_tr[(i * KP + q) * 2], s_tr[(i * KP + q) * 2 + 1]);
  };

  float s[2 * KP];
#pragma unroll UNR
  for (int j = 0; j < 2 * KP; ++j) s[j] = 0.f;

  for (int c = 0; c < nchunk; ++c) {
    const int cn = c + NSTAGE - 1;
    if (cn < nchunk)
      stage_logits<K, NT, TT>(s_stage + (cn % NSTAGE) * NT * P, gbase, LK, cn * T, L, nv, s_len, vec16);
    cp_async_commit();
    cp_async_wait<NSTAGE - 1>();
    __syncthreads();

    const int t0 = c * T;
    if (tid < nv && t0 < mylen) {
      const float* rowp = s_stage + (c % NSTAGE) * NT * P + tid * P;
#pragma unroll
      for (int g = 0; g < T / G; ++g) {
        if (t0 + g * G >= mylen) break;
        float xs[G * K];
        load_group<K>(xs, rowp, g);
#pragma unroll
        for (int gg = 0; gg < G; ++gg) {
          const int t = t0 + g * G + gg;
          if (t < mylen) {
            if (t == 0) {
#pragma unroll UNR
              for (int j = 0; j < K; ++j) s[j] = xs[gg * K + j];
            } else {
              // i-outer order: K independent (best, arg) pairs -> K-way ILP; per (i,j) the fp32 add and the
              // strict '>' (first max wins) are exactly those of the reference recursion
              float best[2 * KP];
              int arg[2 * KP];
#pragma unroll UNR
              for (int q = 0; q < KP; ++q) {
                upk2(add2(pk2(s[0], s[0]), trp(0, q)), best[2 * q], best[2 * q + 1]);
                arg[2 * q] = 0;
                arg[2 * q + 1] = 0;
              }
#pragma unroll UNR
              for (int i = 1; i < K; ++i) {
#pragma unroll UNR
                for (int q = 0; q < KP; ++q) {
                  float lo, hi;
                  upk2(add2(pk2(s[i], s[i]), trp(i, q)), lo, hi);
                  if (lo > best[2 * q]) {
                    best[2 * q] = lo;
                    arg[2 * q] = i;
                  }
                  if (2 * q + 1 < K && hi > best[2 * q + 1]) {
                    best[2 * q + 1] = hi;
                    arg[2 * q + 1] = i;
                  }
                }
              }
              uint32_t wlo = 0u, whi = 0u;
#pragma unroll UNR
              for (int j = 0; j < K; ++j) {
                s[j] = xs[gg * K + j] + best[j];
                if (j < 8)
                  wlo |= (uint32_t)arg[j] << (4 * j);
                else
                  whi |= (uint32_t)arg[j] << (4 * (j - 8));
              }
              __stcg(scratch + (size_t)t * nv + tid, wlo);
              if (HB == 1) s_hi[t * NT + tid] = (uint8_t)whi;
              if (HB == 2) reinterpret_cast<uint16_t*>(s_hi)[t * NT + tid] = (uint16_t)whi;
              if (HB == 4) reinterpret_cast<uint32_t*>(s_hi)[t * NT + tid] = whi;
            }
          }
        }
      }
    }
    __syncthreads();
  }

  if (tid < nv) {
    float best;
    int y = argmax_first<K>(s, best);
    if (best_score != nullptr) best_score[row0 + tid] = best;
    uint8_t* drow = s_dec + tid * Lp;
    // Backtrace: the parked words are at addresses independent of the path, so fetch 8 steps per
    // round trip to L2 and resolve the chain in registers.
    for (int t = mylen - 1; t >= 1; t -= 8) {
      uint32_t wa[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) wa[u] = (t - u >= 1) ? __ldcg(scratch + (size_t)(t - u) * nv + tid) : 0u;
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int tt = t - u;
        if (tt >= 1) {
          uint32_t w = wa[u];
          if (HB > 0 && y >= 8) {
            if (HB == 1) w = s_hi[tt * NT + tid];
            if (HB == 2) w = reinterpret_cast<const uint16_t*>(s_hi)[tt * NT + tid];
            if (HB == 4) w = reinterpret_cast<const uint32_t*>(s_hi)[tt * NT + tid];
          }
          drow[tt] = (uint8_t)y;
          y = (int)((w >> (4 * (y & 7))) & 15u);
        }
      }
    }
    drow[0] = (uint8_t)y;
  }
  __syncthreads();   // every parked word has been consumed: the slab can now take the decoded tags

  store_tags_coalesced<NT>(tags_out + (size_t)row0 * L, nv, L, s_len, [&](int r, int p) { return (int)s_dec[r * Lp + p]; });
}

template <int K, int J = 0, typename F>
__device__ __forceinline__ void sel_all(F& f) {
  if constexpr (J < K) {
    f(std::integral_constant<int, J>{});
    sel_all<K, J + 1>(f);
  }
}

// ---------------------------------------------------------------------------------------------
// Pipe-balanced variant (K <= 16, L*K % 4 == 0): same one-thread-per-sequence decomposition, four changes.
//  (1) The per-(i,j) work of the argmax is split over BOTH arithmetic pipes.  The kernels above spend, per pair, one
//      FADD2 half on the fma pipe and FSETP + FSEL + SEL on the alu pipe: 277 alu vs 60 fma instructions per step at
//      K = 10.  Here the max over i is a tree of max3 (two FMNMX each on sm_90a), and the arg is the
//      FIRST i whose value equals the max: one FSETP.EQ (alu) and one predicated IMAD of a pre-shifted immediate (fma
//      pipe) per pair, walking i downwards so the lowest index is the one that sticks.  That is the reference's strict
//      '>' scan for every non-NaN input (+0 / -0 compare equal in both formulations; the running score may differ in
//      the sign of a zero, never in value).
//  (2) Emission logits arrive by TMA: one cp.async.bulk.tensor per chunk of T steps per warp (box = 32 rows x
//      (T*K + pad) floats of the [B, L*K] view; the pad keeps the row pitch an odd number of 16-byte units so the
//      LDS.128 reads are conflict free; out-of-range columns/rows are zero filled) instead of ~18 instructions per
//      16-byte cp.async request.  Two-stage ring; a stage is refilled as soon as its rows sit in registers, i.e. before
//      the arithmetic of the chunk (an L2 prefetch further ahead measured slower and is not issued).
//  (3) All backpointers stay in shared memory (4 bits per tag: 5 bytes per step at K = 10), so there is no parked
//      traffic to L2/HBM and no 64-bit address arithmetic per step; decoded tags leave in one coalesced sweep.
//  (4) One warp = one CTA = one pipeline (ring, full-barriers, backtrace, output sweep): no CTA barrier in the loop, a
//      warp fetches only to ITS longest row, 8 CTAs per SM.  Chunks that end before the warp's shortest row take a path
//      without per-row length checks; chunk 0 (t = 0 has no predecessor) is peeled.  The backtrace prefetches the words
//      of 8 steps (their addresses do not depend on the path) and resolves the chain in registers.  The transition
//      matrix goes from global memory straight into registers (every thread reads the same K*K words).
// The parked-nibble kernel above serves the calls this one cannot: L*K % 4 != 0, logits not 16-byte aligned, or the
// backpointers of L steps do not fit in shared memory.
template <int K, int TT>
struct TmaGeom {
  static constexpr int T = (K % 2) ? 4 : TT;                // steps per chunk: T*K % 4 == 0
  static constexpr int NQ = T * K / 4;                      // 16-byte units of payload per row-chunk
  static constexpr int PW = 4 * (NQ | 1);                   // row pitch in floats (odd number of 16-byte units)
  static constexpr int KP = (K + 1) / 2;
  static constexpr int HB = BpSplit<K>::HB;
};

template <int K, int NT, int S, int TT>
size_t viterbi_tma_smem_bytes(int L) {
  using Gm = TmaGeom<K, TT>;
  const size_t ring = (size_t)S * NT * Gm::PW * 4;
  const size_t dec = (size_t)NT * (((L + 3) & ~3) + 4);
  const size_t lo = (size_t)L * NT * 4;
  const size_t hi = ((size_t)L * NT * Gm::HB + 15) & ~(size_t)15;
  return (ring > dec ? ring : dec) + lo + hi + (size_t)NT * 4 + 8 + (NT / 32) * S * 8;
}

// ix <- imm where v == m.  Walked from the highest i down, so the lowest equal index is the one that remains.
// The move is written as a predicated multiply-add on the old value with a register that holds 0 (a kernel argument,
// opaque to ptxas): a predicated `mov` becomes SEL and lands on the alu pipe with the compares; the IMAD issues on the
// fma pipe.
#define NER_SEL_EQ(ix, v, m, imm, zero) \
  asm("{\n\t.reg .pred p;\n\tsetp.eq.f32 p, %1, %2;\n\t@p mad.lo.u32 %0, %0, %4, %3;\n\t}" : "+r"(ix) : "f"(v), "f"(m), "n"(imm), "r"(zero))

template <int K, int J>
struct ArgSel {   // compile-time immediates: index i pre-shifted to tag J's nibble
  template <int I>
  static __device__ __forceinline__ void walk(uint32_t& ix, const float* v, float m, uint32_t zero) {
    if constexpr (I >= 0) {
      NER_SEL_EQ(ix, v[I], m, (uint32_t)I << (4 * (J & 7)), zero);
      walk<I - 1>(ix, v, m, zero);
    }
  }
  static __device__ __forceinline__ uint32_t run(const float* v, float m, uint32_t zero) {
    uint32_t ix = (uint32_t)(K - 1) << (4 * (J & 7));
    walk<K - 2>(ix, v, m, zero);
    return ix;
  }
};

// max of v[0..K): three-input maxima over triples, then a three-input tree over those (depth 3 at K = 10)
template <int K>
__device__ __forceinline__ float max_tree(const float* v) {
  if constexpr (K == 1) {
    return v[0];
  } else if constexpr (K == 2) {
    return fmaxf(v[0], v[1]);
  } else if constexpr (K == 3) {
    return max3(v[0], v[1], v[2]);
  } else {
    constexpr int G = (K + 2) / 3;
    float g[G];
#pragma unroll
    for (int a = 0; a < G; ++a) {
      const int n = (3 * a + 3 <= K) ? 3 : (K - 3 * a);
      g[a] = (n == 3) ? max3(v[3 * a], v[3 * a + 1], v[3 * a + 2]) : (n == 2 ? fmaxf(v[3 * a], v[3 * a + 1]) : v[3 * a]);
    }
    return max_tree<G>(g);
  }
}

// One WARP is one independent pipeline: its own TMA ring (box = 32 rows), its own full-barriers, its own backpointer
// columns, backtrace and output sweep; the CTA only carves up shared memory (no CTA barrier after the prologue).
template <int K, int NT, int S, int TT, int MINB>
__global__ void __launch_bounds__(NT, MINB)
crf_viterbi_tma_kernel(const __grid_constant__ CUtensorMap tm_logits, const int32_t* __restrict__ seq_len,
                       const float* __restrict__ trans, int32_t* __restrict__ tags_out,
                       float* __restrict__ best_score, int B, int L, int vec_out, uint32_t zero) {
  using Gm = TmaGeom<K, TT>;
  constexpr int T = Gm::T, PW = Gm::PW, KP = Gm::KP, HB = Gm::HB, NW = NT / 32;
  constexpr uint32_t CHUNK_BYTES = 32 * PW * 4;

  extern __shared__ __align__(128) uint8_t base[];      // the rings come first: TMA destinations stay 16-byte aligned
  const int Lp = ((L + 3) & ~3) + 4;
  const size_t ring_b = (size_t)S * NT * PW * 4, dec_b = (size_t)NT * Lp;
  uint32_t* s_lo = reinterpret_cast<uint32_t*>(base + (ring_b > dec_b ? ring_b : dec_b));   // [L][NT]
  uint8_t* s_hi = reinterpret_cast<uint8_t*>(s_lo + (size_t)L * NT);                // [L][NT] x HB bytes
  int* s_len = reinterpret_cast<int*>(s_hi + (((size_t)L * NT * HB + 15) & ~(size_t)15));     // [NT]
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_len + NT);                         // [NW][S], 8-byte aligned

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);      // provably warp-uniform: ring / barrier addresses stay in uniform registers
  const int row0 = blockIdx.x * NT;
  const int nv = min(NT, B - row0);
  const int wrow0 = row0 + 32 * warp;                   // first row of this warp
  const bool live = tid < nv;
  // the ring and, later, the decoded tags of this warp share one region: the larger of the two per-warp sizes
  const size_t wreg_b = (ring_b > dec_b ? ring_b : dec_b) / NW;
  float* w_ring = reinterpret_cast<float*>(base + warp * wreg_b);                   // [S][32][PW]
  uint8_t* w_dec = base + warp * wreg_b;                                            // [32][Lp] after the forward loop
  uint64_t* w_bar = bars + warp * S;

  if (lane == 0) {
    if (tid == 0) tc::tma_prefetch_desc(&tm_logits);
#pragma unroll
    for (int s = 0; s < S; ++s) tc::mbar_init(w_bar + s, 1);
    tc::fence_barrier_init();
  }
  int mylen = 1;
  if (live) mylen = clamp_len(seq_len, row0 + tid, L);
  s_len[tid] = mylen;
  int wmax = live ? mylen : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
  const int nchunk = (wmax + T - 1) / T;                // 0 for a warp past the end of the batch
  __syncthreads();                                      // s_len and every warp's barrier inits are visible

  if (tc::elect_one()) {
#pragma unroll
    for (int s = 0; s < S; ++s)
      if (s < nchunk) {
        tc::mbar_arrive_expect_tx(w_bar + s, CHUNK_BYTES);
        tc::tma_load_2d(w_ring + (size_t)s * 32 * PW, &tm_logits, w_bar + s, s * T * K, wrow0);
      }
  }

  f32x2 tr2[K * KP];       // tr2[j*KP + p] = (trans[2p][j], trans[2p+1][j]); every thread reads the same K*K words (L1 broadcast)
#pragma unroll
  for (int j = 0; j < K; ++j)
#pragma unroll
    for (int p = 0; p < KP; ++p)
      tr2[j * KP + p] = pk2(__ldg(trans + (2 * p) * K + j), (2 * p + 1 < K) ? __ldg(trans + (2 * p + 1) * K + j) : 0.f);

  f32x2 s2[KP];
#pragma unroll
  for (int p = 0; p < KP; ++p) s2[p] = pk2(0.f, 0.f);

  const int wnv = max(0, min(32, nv - 32 * warp));
  uint32_t* lo_p = s_lo + tid;
  uint8_t* hi_p = s_hi + (size_t)tid * HB;

  int wmin = live ? mylen : L;             // shortest live row of the warp: chunks that end before it need no per-row checks
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) wmin = min(wmin, __shfl_xor_sync(0xffffffffu, wmin, o));

  // one DP step for this lane: s2 <- max-plus(s2, trans) + x_t, backpointers of step t to shared memory
  auto dp_step = [&](const float* xs, const int g, const int t) {
    float m[2 * KP];
    uint32_t wlo = 0u, whi = 0u;
    auto tag_step = [&](auto jc) {
      constexpr int J = decltype(jc)::value;
      float v[2 * KP];
#pragma unroll
      for (int p = 0; p < KP; ++p) upk2(add2(s2[p], tr2[J * KP + p]), v[2 * p], v[2 * p + 1]);
      const float mj = max_tree<K>(v);
      m[J] = mj;
      const uint32_t ix = ArgSel<K, J>::run(v, mj, zero);
      if (J < 8) wlo |= ix; else whi |= ix;
    };
    sel_all<K>(tag_step);
    if (2 * KP > K) m[2 * KP - 1] = 0.f;
#pragma unroll
    for (int p = 0; p < KP; ++p)
      s2[p] = add2(pk2(m[2 * p], m[2 * p + 1]), pk2(xs[g * K + 2 * p], (2 * p + 1 < K) ? xs[g * K + 2 * p + 1] : 0.f));
    lo_p[(size_t)t * NT] = wlo;
    if (HB == 1) hi_p[(size_t)t * NT] = (uint8_t)whi;
    if (HB == 2) reinterpret_cast<uint16_t*>(hi_p)[(size_t)t * NT] = (uint16_t)whi;
    if (HB == 4) reinterpret_cast<uint32_t*>(hi_p)[(size_t)t * NT] = whi;
  };

  // refill of the stage this warp has just copied into registers (warp-uniform condition, one elected lane).  The
  // __syncwarp before it orders every lane's LDS of the stage before the TMA write, the same release the usual
  // consumer-arrive / producer-wait pair gives.
  auto refill = [&](const int c, const int st) {
    __syncwarp();
    if (c + S < nchunk) {
      if (tc::elect_one()) {
        tc::mbar_arrive_expect_tx(w_bar + st, CHUNK_BYTES);
        tc::tma_load_2d(w_ring + (size_t)st * 32 * PW, &tm_logits, w_bar + st, (c + S) * T * K, wrow0);
      }
    }
  };

  auto do_chunk = [&](const int c, auto first_tag) {
    constexpr bool FIRST = decltype(first_tag)::value;       // chunk 0 holds t = 0 (s_0 = x_0, no backpointer)
    const int st = c % S;
    tc::mbar_wait(w_bar + st, (uint32_t)(c / S) & 1u);
    const int t0 = c * T;
    const float4* rowp = reinterpret_cast<const float4*>(w_ring + (size_t)st * 32 * PW + lane * PW);
    if (!FIRST && t0 + T <= wmin) {        // warp-uniform fast path: every live row has all T steps, no per-row checks
      float xs[T * K];
#pragma unroll
      for (int q = 0; q < T * K / 4; ++q) {
        const float4 v = rowp[q];
        xs[4 * q] = v.x; xs[4 * q + 1] = v.y; xs[4 * q + 2] = v.z; xs[4 * q + 3] = v.w;
      }
      refill(c, st);                       // early: the next-but-one chunk is in flight during this chunk's arithmetic
#pragma unroll
      for (int g = 0; g < T; ++g) dp_step(xs, g, t0 + g);
      return;
    }
    if (live && t0 < mylen) {
      float xs[T * K];
#pragma unroll
      for (int q = 0; q < T * K / 4; ++q) {
        const float4 v = rowp[q];
        xs[4 * q] = v.x; xs[4 * q + 1] = v.y; xs[4 * q + 2] = v.z; xs[4 * q + 3] = v.w;
      }
#pragma unroll
      for (int g = 0; g < T; ++g) {
        const int t = t0 + g;
        if (t < mylen) {
          if (FIRST && t == 0) {
#pragma unroll
            for (int p = 0; p < KP; ++p) s2[p] = pk2(xs[2 * p], (2 * p + 1 < K) ? xs[2 * p + 1] : 0.f);
          } else {
            dp_step(xs, g, t);
          }
        }
      }
    }
    refill(c, st);
  };
  if (nchunk > 0) do_chunk(0, std::true_type{});
#pragma unroll 1
  for (int c = 1; c < nchunk; ++c) do_chunk(c, std::false_type{});
  __syncwarp();                            // this warp's ring is dead: its decoded tags may overwrite it

  if (live) {
    float sv[2 * KP];
#pragma unroll
    for (int p = 0; p < KP; ++p) upk2(s2[p], sv[2 * p], sv[2 * p + 1]);
    float best;
    int y = argmax_first<K, true>(sv, best);
    if (best_score != nullptr) best_score[row0 + tid] = best;
    uint8_t* drow = w_dec + lane * Lp;
    // Backtrace: the words are at addresses independent of the path, so fetch 8 steps per round trip and resolve the
    // chain in registers.
    for (int t = mylen - 1; t >= 1; t -= 8) {
      uint32_t wa[8], wb[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const bool in = t - u >= 1;
        wa[u] = in ? lo_p[(size_t)(t - u) * NT] : 0u;
        wb[u] = 0u;
        if (HB == 1) wb[u] = in ? hi_p[(size_t)(t - u) * NT] : 0u;
        if (HB == 2) wb[u] = in ? reinterpret_cast<const uint16_t*>(hi_p)[(size_t)(t - u) * NT] : 0u;
        if (HB == 4) wb[u] = in ? reinterpret_cast<const uint32_t*>(hi_p)[(size_t)(t - u) * NT] : 0u;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int tt = t - u;
        if (tt >= 1) {
          drow[tt] = (uint8_t)y;
          const uint32_t w = (HB > 0 && y >= 8) ? wb[u] : wa[u];
          y = (int)((w >> (4 * (y & 7))) & 15u);
        }
      }
    }
    drow[0] = (uint8_t)y;
  }
  __syncwarp();

  // Coalesced [rows of this warp, L] int32 store; zero beyond each row's length.
  int32_t* obase = tags_out + (size_t)wrow0 * L;
  const int* wlen = s_len + 32 * warp;
  if (vec_out) {
    const int L4 = L >> 2, total4 = wnv * L4;
    int4* o4 = reinterpret_cast<int4*>(obase);
    int r = 0, q = lane;                   // (row, int4 column) of the flat index, kept incrementally: no division
    while (q >= L4) { q -= L4; ++r; }
    for (int idx = lane; idx < total4; idx += 32) {
      const int p = 4 * q;
      const uint32_t pk = *reinterpret_cast<const uint32_t*>(w_dec + r * Lp + p);
      const int n = wlen[r];
      int4 o;
      o.x = (p < n) ? (int)(pk & 255u) : 0;
      o.y = (p + 1 < n) ? (int)((pk >> 8) & 255u) : 0;
      o.z = (p + 2 < n) ? (int)((pk >> 16) & 255u) : 0;
      o.w = (p + 3 < n) ? (int)(pk >> 24) : 0;
      o4[idx] = o;
      q += 32;
      while (q >= L4) { q -= L4; ++r; }
    }
  } else {
    const int total = wnv * L;
    for (int idx = lane; idx < total; idx += 32) {
      const int r = idx / L, p = idx - r * L;
      obase[idx] = (p < wlen[r]) ? (int)w_dec[r * Lp + p] : 0;
    }
  }
}

// Which kernel serves a call: exactly the conditions of the table at the top of this file, in its order.  Pure host
// arithmetic.  `tma_ok` = the logits pointer is 16-byte aligned (and, on the retry in ner_crf_viterbi, the driver
// produced a tensor map).
template <int K>
int viterbi_plan_k(int B, int L, bool tma_ok, int num_sms) {
  const bool lanes_fit = viterbi_lanes_smem_bytes<K>(L) <= kMaxSmem;
  if (B <= NER_CRF_SMALL_B && lanes_fit) return NER_VIT_SMALL;
  // Large batches: 128 sequences per CTA when the backpointer slab fits; small batches
  // spread over more SMs with 32-sequence CTAs.
  const bool big = B > num_sms * 32 * 2;
  if constexpr (K <= 16) {
    if (big && tma_ok && ((size_t)L * K) % 4 == 0 && viterbi_tma_smem_bytes<K, 32, 2, 2>(L) <= kMaxSmem) return NER_VIT_TMA;
    if (big && viterbi_gs_smem_bytes<K, 64, 4>(L) <= kMaxSmem) return NER_VIT_PARKED;
  }
  if (big && viterbi_smem_bytes<K, 128>(L) <= kMaxSmem) return NER_VIT_ONCHIP_128;
  if (viterbi_smem_bytes<K, 32>(L) <= kMaxSmem) return NER_VIT_ONCHIP_32;
  // L past the throughput kernels' on-chip backpointers (document-length batches stacked past NER_CRF_SMALL_B rows): the
  // lane-per-tag kernel keeps 32 + 4*SPW bytes per step on chip and serves any B
  if (B > NER_CRF_SMALL_B && lanes_fit) return NER_VIT_SMALL_ANY_B;
  return NER_VIT_NONE;
}

int viterbi_plan(int B, int L, int K, bool tma_ok, int num_sms) {
#define CALL(KK) return viterbi_plan_k<KK>(B, L, tma_ok, num_sms)
  NER_CRF_DISPATCH_K(K, CALL)
#undef CALL
  return NER_VIT_NONE;
}

// The all-on-chip and parked-nibble kernels take the same arguments and differ in CTA size and shared memory only.
using ThreadPerSeqKernel = void (*)(const float*, const int32_t*, const float*, int32_t*, float*, int, int, int);

int launch_thread_per_seq(ThreadPerSeqKernel kern, int nt, size_t smem, const float* logits, const int32_t* seq_len,
                          const float* trans, int32_t* tags_out, float* best_score, int B, int L, int K, cudaStream_t st) {
  if (smem > kMaxSmem) return NER_ERR_UNSUPPORTED;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  const int vec16 = ((L * K) % 4 == 0) && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0);
  const int grid = (B + nt - 1) / nt;
  kern<<<grid, nt, smem, st>>>(logits, seq_len, trans, tags_out, best_score, B, L, vec16);
  return ner_launch_status();
}

// NER_ERR_UNSUPPORTED = the driver has no cuTensorMapEncodeTiled or refused this map: the caller plans again without TMA.
template <int K, int NT, int S, int TT, int MINB>
int launch_viterbi_tma(const float* logits, const int32_t* seq_len, const float* trans, int32_t* tags_out,
                       float* best_score, int B, int L, cudaStream_t st) {
  using Gm = TmaGeom<K, TT>;
  const size_t LK = (size_t)L * K;
  const size_t smem = viterbi_tma_smem_bytes<K, NT, S, TT>(L);
  tc::EncodeTiledFn fn = tc::tensor_map_encode_fn();
  if (fn == nullptr) return NER_ERR_UNSUPPORTED;
  CUtensorMap map;
  cuuint64_t dims[2] = {(cuuint64_t)LK, (cuuint64_t)B};
  cuuint64_t strides[1] = {(cuuint64_t)LK * 4};
  cuuint32_t box[2] = {(cuuint32_t)Gm::PW, 32u};
  cuuint32_t estr[2] = {1, 1};
  if (fn(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(logits), dims, strides, box, estr,
         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return NER_ERR_UNSUPPORTED;
  auto kern = crf_viterbi_tma_kernel<K, NT, S, TT, MINB>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  const int vec_out = ((L & 3) == 0) && ((reinterpret_cast<uintptr_t>(tags_out) & 15) == 0);
  const int grid = (B + NT - 1) / NT;
  kern<<<grid, NT, smem, st>>>(map, seq_len, trans, tags_out, best_score, B, L, vec_out, 0u);
  return ner_launch_status();
}

// Launch the thread-per-sequence kernel `plan` names (template parameters as in viterbi_plan_k).
template <int K>
int launch_planned(int plan, const float* logits, const int32_t* seq_len, const float* trans, int32_t* tags_out,
                   float* best_score, int B, int L, cudaStream_t st) {
  if constexpr (K <= 16) {
    if (plan == NER_VIT_TMA)
      return launch_viterbi_tma<K, 32, 2, 2, 8>(logits, seq_len, trans, tags_out, best_score, B, L, st);
    if (plan == NER_VIT_PARKED)
      return launch_thread_per_seq(crf_viterbi_gs_kernel<K, 64, 4, 6>, 64, viterbi_gs_smem_bytes<K, 64, 4>(L), logits, seq_len,
                                   trans, tags_out, best_score, B, L, K, st);
  }
  if (plan == NER_VIT_ONCHIP_128)
    return launch_thread_per_seq(crf_viterbi_kernel<K, 128>, 128, viterbi_smem_bytes<K, 128>(L), logits, seq_len, trans,
                                 tags_out, best_score, B, L, K, st);
  if (plan == NER_VIT_ONCHIP_32)
    return launch_thread_per_seq(crf_viterbi_kernel<K, 32>, 32, viterbi_smem_bytes<K, 32>(L), logits, seq_len, trans,
                                 tags_out, best_score, B, L, K, st);
  return NER_ERR_UNSUPPORTED;
}

int run_plan(int plan, const float* logits, const int32_t* seq_len, const float* trans, int32_t* tags_out,
             float* best_score, int B, int L, int K, cudaStream_t st) {
  if (plan == NER_VIT_SMALL || plan == NER_VIT_SMALL_ANY_B)
    return ner_crf_viterbi_small(logits, seq_len, trans, tags_out, best_score, B, L, K, st);
#define CALL(KK) return launch_planned<KK>(plan, logits, seq_len, trans, tags_out, best_score, B, L, st)
  NER_CRF_DISPATCH_K(K, CALL)
#undef CALL
  return NER_ERR_UNSUPPORTED;
}

}  // namespace

extern "C" int ner_crf_viterbi_plan(int B, int L, int K, int logits_aligned, int num_sms) {
  if (B < 1 || L < 1 || K < 1 || K > NER_MAX_TAGS) return NER_VIT_NONE;
  return viterbi_plan(B, L, K, logits_aligned != 0, num_sms);
}

extern "C" int ner_crf_viterbi(const float* logits, const int32_t* seq_len, const float* trans,
                               int32_t* tags_out, float* best_score, int B, int L, int K,
                               ner_stream_t stream) {
  if (B < 0 || L < 1 || K < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!logits || !seq_len || !trans || !tags_out) return NER_ERR_INVALID_ARG;
  if (K > NER_MAX_TAGS) return NER_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int plan = viterbi_plan(B, L, K, (reinterpret_cast<uintptr_t>(logits) & 15) == 0, ner_num_sms());
  int rc = run_plan(plan, logits, seq_len, trans, tags_out, best_score, B, L, K, st);
  // Everything the plan depends on is known before launch, except whether the driver hands out a tensor map: that is
  // the one demotion left at launch time, to the plan computed with TMA excluded.
  if (plan == NER_VIT_TMA && rc == NER_ERR_UNSUPPORTED)
    rc = run_plan(viterbi_plan(B, L, K, false, ner_num_sms()), logits, seq_len, trans, tags_out, best_score, B, L, K, st);
  return rc;
}
