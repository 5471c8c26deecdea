// Partial-annotation CRF log-likelihood and its gradient (Tsuboi et al., COLING 2008), sm_90a.  Row b carries, per
// position t < n_b, a set A_t of allowed tags (bit j of label_mask[b,t], bits >= K ignored):
//     ll_b = logZ_A - logZ,   logZ_A = log sum over the paths with y_t in A_t of exp(score),  logZ the usual partition
//     d ll / d x[t][j]     = P_A(y_t = j) - P(y_t = j)
//     d ll / d trans[i][j] = sum_t P_A(y_{t-1}=i, y_t=j) - P(y_{t-1}=i, y_t=j)
// A one-hot mask is the ordinary CRF; a position allowing all K tags contributes nothing.  The reference has no partial
// CRF, so this definition is not pinned to it (DESIGN.md §3.3).
//
// Both recursions run in one pass over the emissions: alpha_A on the logits with disallowed tags at -inf, alpha on the
// logits as they are.  The two walk the same code, so when nothing is masked they are the same arithmetic and ll is
// exactly 0.0; the backward emits P_A - P per element for the same reason (an all-allowed row's d_logits is exactly 0).
// The constrained fast step takes its max over the allowed tags only: a row whose allowed tags score far below a
// disallowed one would otherwise underflow.  An empty A_t (t < n) makes ll = -inf; the backward treats that row as
// length 0 (zero d_logits, nothing added to d_trans).
//
// Route (a function of the call's shape and flags only, as for crf_loglik.cu / crf_bwd.cu):
//   B <= NER_CRF_SMALL_B  lane per tag (as crf_small.cu), exact logsumexp, forward and backward.  Forward flags bit1
//                         takes the thread-per-sequence kernel instead (tests).
//   forward   thread per sequence; B > 128 * SMs: 64-thread CTAs, 4-step chunks; otherwise 32-thread CTAs, 8-step
//             chunks.  Fast scaled-probability step when the transition matrix spans < 30 nats and is finite, exact
//             per-column logsumexp otherwise or when flags bit0 is set.
//   backward  thread per sequence; 64-thread CTAs when B > 128 * SMs and their staging ring fits in shared memory
//             (K <= 17), 32-thread CTAs otherwise.  Fast / exact as the forward, decided from trans alone.
// The staging, recursion steps, prologues, stores, shared-memory sizes and routes are those of the ordinary loss, in
// crf_common.cuh; the loop bodies here are what differs: two recursions, the allowed-set masks, P_A - P.
// Workspace: alpha_ws [2][B][L][K] = (alpha_A, alpha); logz [B][2] = (logZ_A, logZ).
#include "crf_common.cuh"

namespace {

using namespace crf;

// Does mask m allow none of the K tags?
template <int K>
__device__ __forceinline__ bool mask_empty(unsigned m) {
  return (K < 32 ? (m & ((1u << (K & 31)) - 1u)) : m) == 0u;
}

// The forward state of one recursion: alpha_j = lacc + ln a[j] (fast) or a[j] = alpha_j (exact).
template <int K>
struct Alpha {
  float a[K];
  float lacc;
};

template <int K, int NT, int TT, int MINB>
__global__ void __launch_bounds__(NT, MINB)
crf_partial_fwd_kernel(const float* __restrict__ logits, const int32_t* __restrict__ label_mask,
                       const int32_t* __restrict__ seq_len, const float* __restrict__ trans, float* __restrict__ ll,
                       float* __restrict__ logz_out, float* __restrict__ alpha_ws, int B, int L, int vec_logits,
                       int vec_mask, int force_exact) {
  using Gm = Geom<K, TT>;
  constexpr int T = Gm::T, G = Gm::G, P = Gm::P;
  constexpr int UNR = Gm::UNROLL ? K : 1;

  extern __shared__ __align__(16) float smem[];
  float* s_tr = smem;                                // raw trans [i][j]
  float* s_E = s_tr + Gm::KK4;                       // exp(trans - tmax) [i][j]
  int* s_len = reinterpret_cast<int*>(s_E + Gm::KK4);
  float* s_stage = reinterpret_cast<float*>(s_len + NT);
  int* s_mask = reinterpret_cast<int*>(s_stage + NSTAGE * NT * P);

  const int tid = threadIdx.x;
  const int row0 = blockIdx.x * NT;
  const int nv = min(NT, B - row0);
  const int LK = L * K;

  for (int e = tid; e < K * K; e += NT) s_tr[e] = trans[e];
  int rawlen = 0, mylen = 1;
  if (tid < nv) {
    rawlen = seq_len[row0 + tid];
    mylen = min(max(rawlen, 1), L);
  }
  s_len[tid] = mylen;
  const int bmax = block_max_int<NT>(tid < nv ? mylen : 1, reinterpret_cast<int*>(s_stage));
  float tmax;
  const bool fast = trans_is_narrow(s_tr, K * K, tmax) && !force_exact;
  if (!fast) tmax = 0.f;
  for (int e = tid; e < K * K; e += NT) s_E[e] = fast ? expf(s_tr[e] - tmax) : 0.f;
  __syncthreads();

  const float* gbase = logits + (size_t)row0 * LK;
  const int32_t* mbase = label_mask + (size_t)row0 * L;
  const int nchunk = (bmax + T - 1) / T;

#pragma unroll
  for (int s = 0; s < NSTAGE - 1; ++s) {
    if (s < nchunk) {
      stage_logits<K, NT, TT>(s_stage + s * NT * P, gbase, LK, s * T, L, nv, s_len, vec_logits);
      stage_labels<NT, TT>(s_mask + s * NT * LABP, mbase, L, s * T, nv, s_len, vec_mask);
    }
    cp_async_commit();
  }

  // One step of either recursion.  For the constrained one x holds -inf at the disallowed tags, so the fast path's
  // max is taken over the allowed ones; an empty set leaves xm = -inf, which is replaced by 0 (the row's ll is -inf
  // whatever this step computes).  The fast path renormalises every step.
  auto step = [&](Alpha<K>& s, const float* x, int t) {
    if (fast) {
      float xm = row_max<K>(x);
      if (!(xm > -INFINITY)) xm = 0.f;
      if (t == 0)
        fwd_fast_init<K>(s.a, s.lacc, x, xm);
      else
        fwd_fast_step<K, false>(s.a, s.lacc, x, xm, tmax, nullptr, s_E, true);
    } else if (t == 0) {
#pragma unroll UNR
      for (int j = 0; j < K; ++j) s.a[j] = x[j];
    } else {
      fwd_exact_step<K>(s.a, x, s_tr);
    }
  };

  Alpha<K> sa, sf;  // constrained, free
#pragma unroll UNR
  for (int j = 0; j < K; ++j) sa.a[j] = sf.a[j] = 0.f;
  sa.lacc = sf.lacc = 0.f;
  bool empty = false;  // some A_t (t < len) is empty
  float* aws_a = (alpha_ws != nullptr && tid < nv) ? alpha_ws + (size_t)(row0 + tid) * LK : nullptr;
  float* aws_f = aws_a != nullptr ? aws_a + (size_t)B * LK : nullptr;

  for (int c = 0; c < nchunk; ++c) {
    const int cn = c + NSTAGE - 1;
    if (cn < nchunk) {
      stage_logits<K, NT, TT>(s_stage + (cn % NSTAGE) * NT * P, gbase, LK, cn * T, L, nv, s_len, vec_logits);
      stage_labels<NT, TT>(s_mask + (cn % NSTAGE) * NT * LABP, mbase, L, cn * T, nv, s_len, vec_mask);
    }
    cp_async_commit();
    cp_async_wait<NSTAGE - 1>();
    __syncthreads();

    const int t0 = c * T;
    if (tid < nv && t0 < mylen) {
      const float* rowp = s_stage + (c % NSTAGE) * NT * P + tid * P;
      const int* rowm = s_mask + (c % NSTAGE) * NT * LABP + tid * LABP;
#pragma unroll
      for (int g = 0; g < T / G; ++g) {
        if (t0 + g * G < mylen) {
          float xs[G * K];
          load_group<K>(xs, rowp, g);
#pragma unroll
          for (int gg = 0; gg < G; ++gg) {
            const int tt = g * G + gg;
            const int t = t0 + tt;
            if (t < mylen) {
              const unsigned m = (unsigned)rowm[tt];
              const float* x = xs + gg * K;
              float xa[K];
#pragma unroll UNR
              for (int j = 0; j < K; ++j) xa[j] = ((m >> j) & 1u) ? x[j] : -INFINITY;
              empty |= mask_empty<K>(m);
              step(sa, xa, t);
              step(sf, x, t);
              if (aws_a != nullptr) {
                store_alpha<K>(aws_a + (size_t)t * K, sa.a, sa.lacc, fast);
                store_alpha<K>(aws_f + (size_t)t * K, sf.a, sf.lacc, fast);
              }
            }
          }
        }
      }
    }
    __syncthreads();
  }

  if (tid < nv) {
    float lza = fwd_logz<K>(sa.a, sa.lacc, fast), lzf = fwd_logz<K>(sf.a, sf.lacc, fast);
    if (empty) lza = -INFINITY;
    if (rawlen <= 0) lza = lzf = 0.f;  // empty sequence: ll = 0, nothing to differentiate
    ll[row0 + tid] = lza - lzf;
    if (logz_out != nullptr) {
      logz_out[2 * (row0 + tid)] = lza;
      logz_out[2 * (row0 + tid) + 1] = lzf;
    }
  }
}

template <int K, int NT, int TT, int MINB = 1>
int launch_fwd_nt(const float* logits, const int32_t* mask, const int32_t* seq_len, const float* trans, float* ll,
                  float* logz, float* alpha_ws, int B, int L, int flags, cudaStream_t st) {
  const size_t smem = fwd_smem_bytes<K, NT, TT>();
  auto kern = crf_partial_fwd_kernel<K, NT, TT, MINB>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  const int vl = ((L * K) % 4 == 0) && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0);
  const int vm = (L % 4 == 0) && ((reinterpret_cast<uintptr_t>(mask) & 15) == 0);
  kern<<<(B + NT - 1) / NT, NT, smem, st>>>(logits, mask, seq_len, trans, ll, logz, alpha_ws, B, L, vl, vm, flags & 1);
  return ner_launch_status();
}

template <int K>
int launch_fwd_lanes(const float* logits, const int32_t* mask, const int32_t* seq_len, const float* trans, float* ll,
                     float* logz, float* alpha_ws, int B, int L, cudaStream_t st);

template <int K>
int launch_fwd(const float* logits, const int32_t* mask, const int32_t* seq_len, const float* trans, float* ll,
               float* logz, float* alpha_ws, int B, int L, int flags, cudaStream_t st) {
  if (B <= NER_CRF_SMALL_B && !(flags & 2))  // flags bit1: the throughput kernel at any B (tests)
    return launch_fwd_lanes<K>(logits, mask, seq_len, trans, ll, logz, alpha_ws, B, L, st);
  if (use_cta64(B))
    return launch_fwd_nt<K, 64, 4, 4>(logits, mask, seq_len, trans, ll, logz, alpha_ws, B, L, flags, st);
  return launch_fwd_nt<K, 32, T_CHUNK>(logits, mask, seq_len, trans, ll, logz, alpha_ws, B, L, flags, st);
}

// ---------------------------------------------------------------------------------------------------------- backward

// One reverse pass with beta_A and beta.  Pair marginals (fast path) accumulate per thread as
// acc[i][j] += pa_A[i] q_A[j] - pa[i] q[j]  and are scaled by exp(trans - rowmax) once at the end.
template <int K, int NT>
__global__ void __launch_bounds__(NT)
crf_partial_bwd_kernel(const float* __restrict__ logits, const int32_t* __restrict__ label_mask,
                       const int32_t* __restrict__ seq_len, const float* __restrict__ trans,
                       const float* __restrict__ alpha_ws, const float* __restrict__ logz,
                       const float* __restrict__ d_ll, float scale, float* __restrict__ d_logits,
                       float* __restrict__ d_trans, int B, int L, int vec_logits, int vec_mask) {
  using Gm = Geom<K>;
  constexpr int T = Gm::T, G = Gm::G, P = Gm::P;
  constexpr int UNR = Gm::UNROLL ? K : 1;
  constexpr bool ACC_REGS = Gm::ACC_REGS;

  extern __shared__ __align__(16) float smem[];
  float* s_tr = smem;                                // raw trans [i][j]
  float* s_E = s_tr + Gm::KK4;                       // exp(trans[i][j] - rmax[i])
  float* s_dT = s_E + Gm::KK4;                       // CTA-level d_trans accumulator
  float* s_rmax = s_dT + Gm::KK4;                    // [32]
  int* s_len = reinterpret_cast<int*>(s_rmax + 32);  // [NT]
  float* s_x = reinterpret_cast<float*>(s_len + NT); // [NSTAGE][NT][P] logits, overwritten by d_logits
  float* s_aa = s_x + NSTAGE * NT * P;               // alpha_A
  float* s_af = s_aa + NSTAGE * NT * P;              // alpha
  int* s_mask = reinterpret_cast<int*>(s_af + NSTAGE * NT * P);

  const int tid = threadIdx.x;
  const int row0 = blockIdx.x * NT;
  const int nv = min(NT, B - row0);
  const int LK = L * K;

  float lza = 0.f, lzf = 0.f, gcoef = 0.f;
  int mylen = 0;
  if (tid < nv) {
    mylen = min(max(seq_len[row0 + tid], 0), L);
    lza = logz[2 * (row0 + tid)];
    lzf = logz[2 * (row0 + tid) + 1];
    gcoef = (d_ll != nullptr ? d_ll[row0 + tid] : 1.f) * scale;
    if (!(lza > -INFINITY)) mylen = 0;  // an empty allowed set: ll = -inf, the row adds no gradient
  }
  int bmax;
  const bool fast = bwd_prologue<K, NT>(trans, mylen, s_tr, s_E, s_dT, s_rmax, s_len, reinterpret_cast<int*>(s_x), bmax);

  const float* gx = logits + (size_t)row0 * LK;
  const float* gaa = alpha_ws + (size_t)row0 * LK;
  const float* gaf = gaa + (size_t)B * LK;
  const int32_t* gm = label_mask + (size_t)row0 * L;
  float* gd = d_logits + (size_t)row0 * LK;
  const int nchunk = (bmax + T - 1) / T;
  zero_dlogits_tail<K, NT>(gd, nv, L, nchunk);

  auto stage = [&](int c, int buf) {
    stage_logits<K, NT>(s_x + buf * NT * P, gx, LK, c * T, L, nv, s_len, vec_logits);
    stage_logits<K, NT>(s_aa + buf * NT * P, gaa, LK, c * T, L, nv, s_len, vec_logits);
    stage_logits<K, NT>(s_af + buf * NT * P, gaf, LK, c * T, L, nv, s_len, vec_logits);
    stage_labels<NT>(s_mask + buf * NT * LABP, gm, L, c * T, nv, s_len, vec_mask);
  };
#pragma unroll
  for (int s = 0; s < NSTAGE - 1; ++s) {
    if (s < nchunk) stage(nchunk - 1 - s, s % NSTAGE);
    cp_async_commit();
  }

  // Per recursion: beta, and the step-(t+1) quantities the pair marginal of (t, t+1) needs: q = exp(u - mq) with
  // u = x + beta (fast), or u itself (exact).
  float ba[K], bf[K], qa[K], qf[K], acc[ACC_REGS ? K * K : 1];
  float mqa = 0.f, mqf = 0.f;
#pragma unroll UNR
  for (int j = 0; j < K; ++j) ba[j] = bf[j] = qa[j] = qf[j] = 0.f;
  if constexpr (ACC_REGS) {
#pragma unroll
    for (int e = 0; e < K * K; ++e) acc[e] = 0.f;
  }

  for (int it = 0; it < nchunk; ++it) {
    const int c = nchunk - 1 - it;
    const int itn = it + NSTAGE - 1;
    if (itn < nchunk) stage(nchunk - 1 - itn, itn % NSTAGE);
    cp_async_commit();
    cp_async_wait<NSTAGE - 1>();
    __syncthreads();

    const int buf = it % NSTAGE;
    const int t0 = c * T;
    if (tid < nv && t0 < mylen) {
      float* rowx = s_x + buf * NT * P + tid * P;
      const float* rowaa = s_aa + buf * NT * P + tid * P;
      const float* rowaf = s_af + buf * NT * P + tid * P;
      const int* rowm = s_mask + buf * NT * LABP + tid * LABP;
#pragma unroll
      for (int g = T / G - 1; g >= 0; --g) {
        if (t0 + g * G < mylen) {
          float xs[G * K], aas[G * K], afs[G * K], dl[G * K];
          load_group<K>(xs, rowx, g);
          load_group<K>(aas, rowaa, g);
          load_group<K>(afs, rowaf, g);
#pragma unroll
          for (int gg = G - 1; gg >= 0; --gg) {
            const int tt = g * G + gg;
            const int t = t0 + tt;
            if (t < mylen) {
              const float* aa = aas + gg * K;
              const float* af = afs + gg * K;
              // ---- pair marginals of (t, t+1) from step t+1's q / mq
              if (t < mylen - 1) {
                if (fast) {
                  float pa[K], pf[K];
#pragma unroll UNR
                  for (int i = 0; i < K; ++i) {
                    pa[i] = __expf(aa[i] + s_rmax[i] + mqa - lza);
                    pf[i] = __expf(af[i] + s_rmax[i] + mqf - lzf);
                  }
                  if constexpr (ACC_REGS) {
#pragma unroll
                    for (int i = 0; i < K; ++i)
#pragma unroll
                      for (int j = 0; j < K; ++j) acc[i * K + j] += __fmul_rn(pa[i], qa[j]) - __fmul_rn(pf[i], qf[j]);
                  } else {
                    for (int i = 0; i < K; ++i)
                      for (int j = 0; j < K; ++j) {
                        const float d = __fmul_rn(pa[i], qa[j]) - __fmul_rn(pf[i], qf[j]);
                        if (d != 0.f) atomicAdd(&s_dT[i * K + j], gcoef * d * s_E[i * K + j]);
                      }
                  }
                } else {
                  for (int i = 0; i < K; ++i)
                    for (int j = 0; j < K; ++j) {
                      const float d = expf(aa[i] + s_tr[i * K + j] + qa[j] - lza) -
                                      expf(af[i] + s_tr[i * K + j] + qf[j] - lzf);
                      if (d != 0.f) atomicAdd(&s_dT[i * K + j], gcoef * d);
                    }
                }
              }
              // ---- unary marginals: d_logits = g (P_A - P), an exact +0 where they agree
#pragma unroll UNR
              for (int j = 0; j < K; ++j) {
                const float d = __expf(aa[j] + ba[j] - lza) - __expf(af[j] + bf[j] - lzf);
                dl[gg * K + j] = fmaf(gcoef, d, 0.f);
              }
              // ---- beta recursions to t-1
              if (t > 0) {
                const unsigned m = (unsigned)rowm[tt];
                const float* x = xs + gg * K;
                float ua[K], uf[K];
#pragma unroll UNR
                for (int j = 0; j < K; ++j) {
                  uf[j] = x[j] + bf[j];
                  ua[j] = ((m >> j) & 1u) ? x[j] + ba[j] : -INFINITY;
                }
                beta_step<K>(fast, ba, qa, mqa, qa, ua, s_tr, s_E, s_rmax);
                beta_step<K>(fast, bf, qf, mqf, qf, uf, s_tr, s_E, s_rmax);
              }
            } else {
#pragma unroll UNR
              for (int j = 0; j < K; ++j) dl[gg * K + j] = 0.f;
            }
          }
          float4* o4 = reinterpret_cast<float4*>(rowx + g * G * K);
#pragma unroll
          for (int qq = 0; qq < Gm::GQ; ++qq)
            o4[qq] = make_float4(dl[4 * qq], dl[4 * qq + 1], dl[4 * qq + 2], dl[4 * qq + 3]);
        }
      }
    }
    __syncthreads();
    store_dlogits_chunk<K, NT>(gd, s_x + buf * NT * P, s_len, nv, L, t0, vec_logits);
    __syncthreads();
  }

  flush_dtrans<K, NT>(acc, gcoef, tid < nv, s_dT, s_E, d_trans);
}

template <int K, int NT>
int launch_bwd_nt(const float* logits, const int32_t* mask, const int32_t* seq_len, const float* trans,
                  const float* alpha_ws, const float* logz, const float* d_ll, float scale, float* d_logits,
                  float* d_trans, int B, int L, cudaStream_t st) {
  const size_t smem = bwd_smem_bytes<K, NT, 3>();
  auto kern = crf_partial_bwd_kernel<K, NT>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  const int vl = ((L * K) % 4 == 0) && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0) &&
                 ((reinterpret_cast<uintptr_t>(alpha_ws) & 15) == 0) &&
                 ((reinterpret_cast<uintptr_t>(d_logits) & 15) == 0);
  const int vm = (L % 4 == 0) && ((reinterpret_cast<uintptr_t>(mask) & 15) == 0);
  kern<<<(B + NT - 1) / NT, NT, smem, st>>>(logits, mask, seq_len, trans, alpha_ws, logz, d_ll, scale, d_logits, d_trans,
                                            B, L, vl, vm);
  return ner_launch_status();
}

// ------------------------------------------------------------------------------------- small batches: lane per tag
// B <= NER_CRF_SMALL_B.  The lane-per-tag scheme of crf_small.cu: a group of GS lanes holds one sequence, lane j owns
// tag j of both recursions, predecessors are exchanged with __shfl_sync, every logsumexp is exact with its own max.
// The constrained and the free recursion run the same instructions on x_A and x, so a row with every tag allowed stays
// exactly 0 here too.

template <int K>
__global__ void __launch_bounds__(32)
crf_partial_fwd_lanes_kernel(const float* __restrict__ logits, const int32_t* __restrict__ label_mask,
                             const int32_t* __restrict__ seq_len, const float* __restrict__ trans,
                             float* __restrict__ ll, float* __restrict__ logz_out, float* __restrict__ alpha_ws, int B,
                             int L) {
  constexpr int GS = Lanes<K>::GS, SPW = Lanes<K>::SPW, PF = 4;
  __shared__ float s_tr[K * K];
  const int lane = threadIdx.x;
  const int g = lane / GS, j = lane % GS;
  const int b = blockIdx.x * SPW + g;
  const bool seq_ok = b < B;
  const bool tag_ok = j < K;
  for (int e = lane; e < K * K; e += 32) s_tr[e] = trans[e];
  int rawlen = 0, len = 1;
  if (seq_ok) {
    rawlen = seq_len[b];
    len = min(max(rawlen, 1), L);
  }
  const int wmax = lanes_wmax(len);
  __syncwarp();
  float tc[K];
#pragma unroll
  for (int i = 0; i < K; ++i) tc[i] = tag_ok ? s_tr[i * K + j] : 0.f;

  const size_t base = (size_t)(seq_ok ? b : 0) * L;
  const float* xp = logits + base * K + (tag_ok ? j : 0);
  const int32_t* mp = label_mask + base;
  float* wa = (alpha_ws != nullptr && seq_ok && tag_ok) ? alpha_ws + base * K + j : nullptr;
  float* wf = wa != nullptr ? wa + (size_t)B * L * K : nullptr;
  auto ld = [&](int t) -> float { return (seq_ok && tag_ok && t < len) ? xp[(size_t)t * K] : -INFINITY; };
  auto ldm = [&](int t) -> unsigned { return (seq_ok && t < len) ? (unsigned)mp[t] : 0u; };

  float af = ld(0);
  unsigned m0 = ldm(0);
  float aa = ((m0 >> j) & 1u) ? af : -INFINITY;
  bool empty = mask_empty<K>(m0);
  if (wa != nullptr) {
    wa[0] = aa;
    wf[0] = af;
  }
  float xq[PF];
  unsigned mq[PF];
#pragma unroll
  for (int u = 0; u < PF; ++u) {
    xq[u] = ld(1 + u);
    mq[u] = ldm(1 + u);
  }
  for (int t0 = 1; t0 < wmax; t0 += PF) {
#pragma unroll
    for (int u = 0; u < PF; ++u) {
      const int t = t0 + u;
      const float x = xq[u];
      const unsigned m = mq[u];
      xq[u] = ld(t + PF);
      mq[u] = ldm(t + PF);
      if (t < wmax) {
        const float nf = lanes_alpha_step<K>(af, x, tc, g);
        const float na = lanes_alpha_step<K>(aa, ((m >> j) & 1u) ? x : -INFINITY, tc, g);
        if (t < len) {
          af = tag_ok ? nf : -INFINITY;
          aa = tag_ok ? na : -INFINITY;
          empty |= mask_empty<K>(m);
          if (wa != nullptr) {
            wa[(size_t)t * K] = aa;
            wf[(size_t)t * K] = af;
          }
        }
      }
    }
  }
  float lza = lanes_logsumexp<K>(aa, tag_ok), lzf = lanes_logsumexp<K>(af, tag_ok);
  if (j == 0 && seq_ok) {
    if (empty) lza = -INFINITY;
    if (rawlen <= 0) lza = lzf = 0.f;
    ll[b] = lza - lzf;
    if (logz_out != nullptr) {
      logz_out[2 * b] = lza;
      logz_out[2 * b + 1] = lzf;
    }
  }
}

// Lane i = tag i walks t = len-1 .. 0 with beta_A[i] and beta[i]:
//   w_j = x_t[j] + beta_t[j] (w_A: -inf where tag j is not allowed at t),  v_ij = trans[i][j] + w_j,
//   beta_{t-1}[i] = logsumexp_j v_ij,  pair (t-1, t): exp(alpha_{t-1}[i] - logZ + v_ij),
//   d_x[t][i] = g (exp(alpha_A,t[i] + beta_A,t[i] - logZ_A) - exp(alpha_t[i] + beta_t[i] - logZ)).
template <int K>
__global__ void __launch_bounds__(32)
crf_partial_bwd_lanes_kernel(const float* __restrict__ logits, const int32_t* __restrict__ label_mask,
                             const int32_t* __restrict__ seq_len, const float* __restrict__ trans,
                             const float* __restrict__ alpha_ws, const float* __restrict__ logz,
                             const float* __restrict__ d_ll, float scale, float* __restrict__ d_logits,
                             float* __restrict__ d_trans, int B, int L) {
  constexpr int GS = Lanes<K>::GS, SPW = Lanes<K>::SPW, PF = 4;
  const int lane = threadIdx.x;
  const int g = lane / GS, i = lane % GS;
  const int b = blockIdx.x * SPW + g;
  const bool seq_ok = b < B;
  const bool tag_ok = i < K;
  int len = 0;
  float lza = 0.f, lzf = 0.f, gco = 0.f;
  if (seq_ok) {
    len = min(max(seq_len[b], 0), L);
    lza = logz[2 * b];
    lzf = logz[2 * b + 1];
    gco = (d_ll != nullptr ? d_ll[b] : 1.f) * scale;
    if (!(lza > -INFINITY)) len = 0;  // no path inside the sets: ll = -inf, the row adds no gradient
  }
  const int wmax = lanes_wmax(len);

  float tr[K], acc[K];
#pragma unroll
  for (int jj = 0; jj < K; ++jj) {
    tr[jj] = tag_ok ? trans[i * K + jj] : 0.f;
    acc[jj] = 0.f;
  }
  const size_t base = (size_t)(seq_ok ? b : 0) * L;
  const bool io = seq_ok && tag_ok;
  const float* xp = logits + base * K + (tag_ok ? i : 0);
  const float* pa = alpha_ws + base * K + (tag_ok ? i : 0);
  const float* pf = pa + (size_t)B * L * K;
  const int32_t* mp = label_mask + base;
  float* dp = d_logits + base * K + (tag_ok ? i : 0);
  if (io)
    for (int t = len; t < L; ++t) dp[(size_t)t * K] = 0.f;
  auto ldx = [&](int t) -> float { return (io && t >= 0 && t < len) ? xp[(size_t)t * K] : 0.f; };
  auto lda = [&](const float* p, int t) -> float { return (io && t >= 0 && t < len) ? p[(size_t)t * K] : 0.f; };
  auto ldm = [&](int t) -> unsigned { return (seq_ok && t >= 0 && t < len) ? (unsigned)mp[t] : 0u; };

  float ba = 0.f, bf = 0.f;
  float xq[PF], aaq[PF], afq[PF];
  unsigned mq[PF];
#pragma unroll
  for (int u = 0; u < PF; ++u) {
    xq[u] = ldx(len - 1 - u);
    mq[u] = ldm(len - 1 - u);
    aaq[u] = lda(pa, len - 2 - u);
    afq[u] = lda(pf, len - 2 - u);
  }
  float aa_t = lda(pa, len - 1), af_t = lda(pf, len - 1);
  for (int s0 = 0; s0 < wmax; s0 += PF) {
#pragma unroll
    for (int u = 0; u < PF; ++u) {
      const int sidx = s0 + u;
      const int t = len - 1 - sidx;
      const float x = xq[u], aa_prev = aaq[u], af_prev = afq[u];
      const unsigned m = mq[u];
      xq[u] = ldx(t - PF);
      mq[u] = ldm(t - PF);
      aaq[u] = lda(pa, t - 1 - PF);
      afq[u] = lda(pf, t - 1 - PF);
      if (sidx < wmax) {                    // warp-uniform: every lane takes part in the shuffles
        const bool live = t >= 0;
        if (io && live) dp[(size_t)t * K] = fmaf(gco, __expf(aa_t + ba - lza) - __expf(af_t + bf - lzf), 0.f);
        const float wf_ = (tag_ok && live) ? x + bf : -INFINITY;
        const float wa_ = (tag_ok && live && ((m >> i) & 1u)) ? x + ba : -INFINITY;
        float vf[K], va[K];
        const float mf = lanes_gather<K>(vf, wf_, tr, g);
        const float ma = lanes_gather<K>(va, wa_, tr, g);
        if (live && t >= 1) {
          const float mmf = (fabsf(mf) <= 3.0e38f) ? mf : 0.f;
          const float mma = (fabsf(ma) <= 3.0e38f) ? ma : 0.f;
          const float amf = af_prev - lzf, ama = aa_prev - lza;
          float sf = 0.f, sa = 0.f;
#pragma unroll
          for (int jj = 0; jj < K; ++jj) {
            sf += __expf(vf[jj] - mmf);
            sa += __expf(va[jj] - mma);
            acc[jj] += __expf(ama + va[jj]) - __expf(amf + vf[jj]);
          }
          bf = __logf(sf) + mmf;
          ba = __logf(sa) + mma;
          af_t = af_prev;
          aa_t = aa_prev;
        }
      }
    }
  }
  if (io && len > 0) {
#pragma unroll
    for (int jj = 0; jj < K; ++jj)
      if (acc[jj] != 0.f) atomicAdd(d_trans + i * K + jj, gco * acc[jj]);
  }
}

template <int K>
int launch_fwd_lanes(const float* logits, const int32_t* mask, const int32_t* seq_len, const float* trans, float* ll,
                     float* logz, float* alpha_ws, int B, int L, cudaStream_t st) {
  constexpr int SPW = Lanes<K>::SPW;
  crf_partial_fwd_lanes_kernel<K><<<(B + SPW - 1) / SPW, 32, 0, st>>>(logits, mask, seq_len, trans, ll, logz, alpha_ws,
                                                                      B, L);
  return ner_launch_status();
}

template <int K>
int launch_bwd_lanes(const float* logits, const int32_t* mask, const int32_t* seq_len, const float* trans,
                     const float* alpha_ws, const float* logz, const float* d_ll, float scale, float* d_logits,
                     float* d_trans, int B, int L, cudaStream_t st) {
  constexpr int SPW = Lanes<K>::SPW;
  crf_partial_bwd_lanes_kernel<K><<<(B + SPW - 1) / SPW, 32, 0, st>>>(logits, mask, seq_len, trans, alpha_ws, logz,
                                                                      d_ll, scale, d_logits, d_trans, B, L);
  return ner_launch_status();
}

template <int K>
int launch_bwd(const float* logits, const int32_t* mask, const int32_t* seq_len, const float* trans,
               const float* alpha_ws, const float* logz, const float* d_ll, float scale, float* d_logits,
               float* d_trans, int B, int L, cudaStream_t st) {
  if (B <= NER_CRF_SMALL_B)
    return launch_bwd_lanes<K>(logits, mask, seq_len, trans, alpha_ws, logz, d_ll, scale, d_logits, d_trans, B, L, st);
  // 64-thread CTAs need a three-tensor staging ring twice as large: only up to K = 17 does it fit
  if constexpr (bwd_smem_bytes<K, 64, 3>() <= kMaxSmem) {
    if (use_cta64(B))
      return launch_bwd_nt<K, 64>(logits, mask, seq_len, trans, alpha_ws, logz, d_ll, scale, d_logits, d_trans, B, L,
                                  st);
  }
  return launch_bwd_nt<K, 32>(logits, mask, seq_len, trans, alpha_ws, logz, d_ll, scale, d_logits, d_trans, B, L, st);
}

}  // namespace

extern "C" int ner_crf_partial_loglik_fwd(const float* logits, const int32_t* label_mask, const int32_t* seq_len,
                                          const float* trans, float* ll, float* logz, float* alpha_ws, int B, int L,
                                          int K, int flags, ner_stream_t stream) {
  if (B < 0 || L < 1 || K < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!logits || !label_mask || !seq_len || !trans || !ll) return NER_ERR_INVALID_ARG;
  if (K > NER_MAX_TAGS) return NER_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define CALL(KK) return launch_fwd<KK>(logits, label_mask, seq_len, trans, ll, logz, alpha_ws, B, L, flags, st)
  NER_CRF_DISPATCH_K(K, CALL)
#undef CALL
  return NER_ERR_UNSUPPORTED;
}

extern "C" int ner_crf_partial_loglik_bwd(const float* logits, const int32_t* label_mask, const int32_t* seq_len,
                                          const float* trans, const float* alpha_ws, const float* logz,
                                          const float* d_ll, float scale, float* d_logits, float* d_trans, int B,
                                          int L, int K, ner_stream_t stream) {
  if (B < 0 || L < 1 || K < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!logits || !label_mask || !seq_len || !trans || !alpha_ws || !logz || !d_logits || !d_trans)
    return NER_ERR_INVALID_ARG;
  if (K > NER_MAX_TAGS) return NER_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define CALL(KK) \
  return launch_bwd<KK>(logits, label_mask, seq_len, trans, alpha_ws, logz, d_ll, scale, d_logits, d_trans, B, L, st)
  NER_CRF_DISPATCH_K(K, CALL)
#undef CALL
  return NER_ERR_UNSUPPORTED;
}
