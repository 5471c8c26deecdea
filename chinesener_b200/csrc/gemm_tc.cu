// Dense layers of the encoder on the Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a.
//
//   out[M,N] = epilogue( A[M,K] · Wt[N,K]^T + bias[N] )       A, Wt bf16 (K-major), fp32 accumulate
//
// Replaces the tf.layers.dense / BertModel dense_layer matmuls executed inside
// reference tools/layer.py:68-77 (bert_base.bert.modeling) and model/bert_bilstm_crf.py:26,
// and the input projection half of the LSTMCell matmul (tools/layer.py:16,35).
//
// Kernel shape (persistent, warp-specialised, 384 threads = 3 warpgroups, 1 CTA/SM):
//   warpgroup 0    TMA producer : one elected thread issues cp.async.bulk.tensor 2-D loads of a 128x64 A box and a
//                                 BN x 64 B box per k-block into a STAGES-deep smem ring (SWIZZLE_128B), mbarrier tx;
//                                 it gives its registers to the MMA warpgroups (setmaxnreg)
//   warpgroups 1-2 MMA + epilogue: warpgroup w owns rows 64(w-1) .. 64(w-1)+63 of the tile; per k-block four
//                                 wgmma.m64nBNk16 from SWIZZLE_128B descriptors, fp32 accumulator in registers, one
//                                 wgmma group kept in flight before the previous smem slot is released; then bias /
//                                 GELU / residual in registers, the slice written in 8 KB column chunks (64 bf16 or
//                                 32 fp32 columns x 64 rows) to a double-buffered SWIZZLE_128B staging buffer and
//                                 stored by TMA (cp.async.bulk.tensor, bulk groups).  The warpgroup goes on to the
//                                 next tile's k-blocks while the stores drain; TMA clips the M tail and N past the end.
// While the MMA warpgroups run the epilogue of tile i the producer already fills the ring for tile i+1.
//
// Variants (EPI = the NER_EPI_* mode, a template parameter: no per-element mode test):
//   gemm_bf16_tc_kernel<BN, SK, 1, EPI>   128 x BN tile per CTA (BN = 64/128/192/256), optionally stream-K
//   gemm_bf16_tc_kernel<BN, 0, 2, EPI>    a cluster of 2 CTAs computes a 256 x BN tile: each CTA stages its own 128 A
//                                         rows and loads HALF of the B tile with TMA multicast into both CTAs, so the
//                                         L2->smem bytes per FLOP drop by 1.5x vs the 128 x BN single-CTA tile.
#include <stdlib.h>

#include <mutex>

#include "tc_common.cuh"

namespace {

using namespace tc;

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle-128B row
constexpr int MMA_K = 16;
constexpr int NUM_MMA_WG = 2;
// stream-K fixed charge in k-block times: parking + re-reading a 128 x 256 fp32 partial accumulator and the
// exposed finisher epilogue; it pays when tiles << SMs and K is long (weight gradients, K = tokens).
constexpr float kSkFixupCost = 10.0f;
constexpr int NUM_THREADS = 128 * (1 + NUM_MMA_WG);

// Output staging: per MMA warpgroup two 8 KB chunk buffers (64 rows of 128 B), so a chunk is written while the TMA store
// of the previous one still reads its buffer.
constexpr int OUT_CHUNK_BYTES = 64 * 128;
constexpr int OUT_STAGE_BYTES = NUM_MMA_WG * 2 * OUT_CHUNK_BYTES;

template <int BN>
struct Cfg {
  // 227 KB of shared memory per block = ring + 32 KB output staging + barriers:
  // 4 x 48 KB (BN 256), 4 x 40 KB (192: five stages would not leave room for the staging), 6 x 32 KB (128), 8 x 24 KB (64)
  static constexpr int STAGES = (BN == 256 || BN == 192) ? 4 : ((BN == 128) ? 6 : 8);
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int RING_BYTES = STAGES * (A_BYTES + B_BYTES);
  // ring + staging + barriers; the dynamic smem base is 1024-aligned (checked in-kernel)
  static constexpr size_t SMEM = (size_t)RING_BYTES + OUT_STAGE_BYTES + 256;
  static_assert(SMEM <= 227 * 1024, "shared memory per block");
};

struct EpiArgs {
  const float* bias;      // [N] or null
  const float* residual;  // [M,N] fp32 or null (EPI_RES_F32 / EPI_RES_RELU_F32)
};

template <int EPI>
__host__ __device__ constexpr bool epi_f32() { return EPI == NER_EPI_F32 || EPI == NER_EPI_RES_F32 || EPI == NER_EPI_RES_RELU_F32; }

__device__ __forceinline__ float gelu_tanh(float x) {
  // 0.5x(1+tanh(sqrt(2/pi)(x+0.044715x^3)))  (google-research/bert modeling.gelu).
  // tanh.approx.f32 is one MUFU op (rel. error ~2^-11); the result is rounded to bf16 (2^-9).
  const float u = 0.7978845608028654f * fmaf(0.044715f * x * x, x, x);
  const float hx = 0.5f * x;
  return fmaf(hx, tanh_approx(u), hx);
}
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.7071067811865476f)); }

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

// ---------------------------------------------------------------------------------------------
// Stream-K work split.  With SK the M x N x K iteration space is cut into tiles * num_kb k-block
// units and CTA c owns the contiguous unit range [c*U/G, (c+1)*U/G): every SM gets the same number
// of k-blocks whatever tiles/SMs is (the packed M of an MSRA batch gives fractional waves on
// the encoder's GEMMs, i.e. idle SMs with whole-tile scheduling).  A CTA's range is
//   [tail piece of a tile]  [whole tiles]  [head piece of a tile]
// The CTA holding a tile's HEAD (kb0 == 0) finishes that tile: it adds the fp32 partial sums that
// the CTAs holding the later k-blocks parked in their workspace slot and runs the normal epilogue.
// A tail piece is always the FIRST thing its CTA does and the head piece the LAST, so a finisher
// never waits in practice and no wait cycle can form (all CTAs are co-resident: grid <= #SMs).
struct SkArgs {
  float4* ws;   // [grid][128 x 256 floats]: slot c = partial accumulator of CTA c's first segment
  int* flags;   // [grid] 0 / 1 = slot c published; reset to 0 by the finisher (all zero between launches)
};

// Work iterator over tiles (whole-tile round robin) or stream-K unit ranges; `id` / `count` = this CTA (or CTA
// pair) and the number of them.
struct SegIter {
  int num_kb, num_tiles, tile, stride;
  long long u, u1;
  bool sk;
  __device__ SegIter(bool sk_, int num_tiles_, int num_kb_, int id, int count)
      : num_kb(num_kb_), num_tiles(num_tiles_), sk(sk_) {
    if (sk) {
      const long long U = (long long)num_tiles * num_kb;
      u = (long long)id * U / count;
      u1 = (long long)(id + 1) * U / count;
    } else {
      tile = id;
      stride = count;
    }
  }
  __device__ bool next(int& t, int& kb0, int& kb1) {
    if (sk) {
      if (u >= u1) return false;
      t = (int)(u / num_kb);
      kb0 = (int)(u - (long long)t * num_kb);
      const long long rem = u1 - u;
      kb1 = (rem < (long long)(num_kb - kb0)) ? kb0 + (int)rem : num_kb;
      u += kb1 - kb0;
      return true;
    }
    if (tile >= num_tiles) return false;
    t = tile;
    kb0 = 0;
    kb1 = num_kb;
    tile += stride;
    return true;
  }
};

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__device__ __forceinline__ void mma_bar_sync() {  // named barrier 1 over the MMA warpgroups only
  asm volatile("bar.sync 1, %0;" ::"n"(128 * NUM_MMA_WG) : "memory");
}

// Shared-memory ring of one CTA: STAGES slots of {A tile, B tile}, a `full` barrier per slot (TMA transaction
// bytes) and an `empty` barrier per slot (one arrive per MMA warp of every CTA that reads the slot's bytes).
template <int BN>
struct Ring {
  uint8_t* a;
  uint8_t* b;
  uint8_t* out;   // output staging, OUT_STAGE_BYTES (1024-aligned)
  uint64_t* full;
  uint64_t* empty;
  __device__ Ring(uint8_t* smem) {
    using C = Cfg<BN>;
    a = smem;
    b = smem + C::STAGES * C::A_BYTES;
    out = smem + C::RING_BYTES;
    full = reinterpret_cast<uint64_t*>(out + OUT_STAGE_BYTES);
    empty = full + C::STAGES;
  }
};

struct RingPos {
  int stage = 0;
  uint32_t phase = 0;
  template <int STAGES>
  __device__ __forceinline__ void advance() {
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1u;
    }
  }
};

// MMA side of k-blocks [kb0, kb1): this warpgroup's 64 x BN slice of the tile into `acc`.  A and B descriptors for a
// K-step of 16 are produced by `desc_a(addr, k)` / `desc_b(addr, k)`; TA / TB = operand is MN-major.  The smem slot of
// k-block i is released once the wgmma group of k-block i+1 is issued and group i has retired.
template <int BN, int STAGES, int CL, int TA, int TB, typename DA, typename DB>
__device__ __forceinline__ void mma_kblocks(float (&acc)[BN / 2], const Ring<BN>& ring, RingPos& pos, int kb0, int kb1,
                                            uint32_t a_off, DA desc_a, DB desc_b, const uint32_t (&empty_peer)[STAGES]) {
  const int lane = threadIdx.x & 31;
  int prev = -1;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&ring.full[pos.stage], pos.phase);
    const uint32_t a_addr = smem_u32(ring.a + pos.stage * (BM * BK * 2)) + a_off;
    const uint32_t b_addr = smem_u32(ring.b + pos.stage * (BN * BK * 2));
    reg_fence(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / MMA_K; ++k)
      wgmma_bf16<BN, TA, TB>(acc, desc_a(a_addr, k), desc_b(b_addr, k), (kb > kb0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    reg_fence(acc);
    if (prev >= 0) {
      wgmma_wait<1>();
      reg_fence(acc);
      if (lane == 0) {
        mbar_arrive(&ring.empty[prev]);
        if constexpr (CL == 2) mbar_arrive_cluster(empty_peer[prev]);
      }
    }
    prev = pos.stage;
    pos.template advance<STAGES>();
  }
  wgmma_wait<0>();
  reg_fence(acc);
  if (lane == 0 && prev >= 0) {
    mbar_arrive(&ring.empty[prev]);
    if constexpr (CL == 2) mbar_arrive_cluster(empty_peer[prev]);
  }
}

// Activation of the epilogue, applied after bias (and residual) are added.
template <int EPI>
__device__ __forceinline__ float epi_act(float v) {
  if constexpr (EPI == NER_EPI_GELU_TANH_BF16) return gelu_tanh(v);
  else if constexpr (EPI == NER_EPI_GELU_ERF_BF16) return gelu_erf(v);
  else if constexpr (EPI == NER_EPI_RELU_BF16 || EPI == NER_EPI_RES_RELU_F32) return fmaxf(v, 0.f);
  else return v;
}

__device__ __forceinline__ void wg_bar_sync(int id) {  // named barrier `id` over the 128 threads of one warpgroup
  asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory");
}

// Fused epilogue of one MMA warpgroup's 64 x BN slice (rows row_wg .., columns n0 ..) through shared memory and TMA.
// Thread fragment: rows r, r + 8 (r = 16 warp + lane / 4), column pairs 8 j + 2 (lane % 4).  Chunk c of the slice (CW
// columns, 64 rows, 128-B rows in the SWIZZLE_128B layout the store's tensor map expects: 16-B unit u of row r sits at
// unit u ^ (r % 8)) is written into staging buffer `buf`, then one thread issues its TMA store as one bulk group.  A
// buffer is rewritten only after the store issued from it two chunks earlier has finished reading it.
template <int BN, int EPI>
__device__ __forceinline__ void epilogue_tma(const float (&acc)[BN / 2], const EpiArgs& ep, const CUtensorMap* tma_out,
                                             uint8_t* stage, uint32_t& buf, int row_wg, int n0, int M, int N) {
  constexpr bool F32 = epi_f32<EPI>();
  constexpr bool RES = EPI == NER_EPI_RES_F32 || EPI == NER_EPI_RES_RELU_F32;
  constexpr int CW = F32 ? 32 : 64;   // columns per 8 KB chunk
  constexpr int JPC = CW / 8;         // fragment column groups per chunk
  const int t = threadIdx.x & 127, lane = t & 31, warp = t >> 5;
  const int bar = 1 + (threadIdx.x >> 7);   // 2, 3 (1 = both MMA warpgroups)
  const int r0 = 16 * warp + (lane >> 2);
  if (row_wg >= M) return;   // the whole slice lies past M (tail of a 2-CTA tile)
#pragma unroll
  for (int c = 0; c < BN / CW; ++c) {
    const int col0 = n0 + c * CW;
    if (col0 >= N) break;
    uint8_t* sb = stage + buf * OUT_CHUNK_BYTES;
    if (t == 0) tma_store_wait_read<1>();
    wg_bar_sync(bar);
    float2 b[JPC];
#pragma unroll
    for (int jj = 0; jj < JPC; ++jj) {
      const int col = col0 + 8 * jj + 2 * (lane & 3);
      b[jj] = (ep.bias != nullptr && col < N) ? __ldg(reinterpret_cast<const float2*>(ep.bias + col)) : make_float2(0.f, 0.f);
    }
    if constexpr (F32) {
#pragma unroll
      for (int jj = 0; jj < JPC; ++jj) {
        const int j = c * JPC + jj, col = col0 + 8 * jj + 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = r0 + 8 * h;
          float v0 = acc[4 * j + 2 * h] + b[jj].x, v1 = acc[4 * j + 2 * h + 1] + b[jj].y;
          if constexpr (RES) {
            const int row = row_wg + r;
            if (row < M && col < N) {
              const float2 rv = *reinterpret_cast<const float2*>(ep.residual + (size_t)row * N + col);
              v0 += rv.x;
              v1 += rv.y;
            }
          }
          v0 = epi_act<EPI>(v0);
          v1 = epi_act<EPI>(v1);
          const int unit = (2 * jj + ((lane & 3) >> 1)) ^ (r & 7);
          *reinterpret_cast<float2*>(sb + r * 128 + unit * 16 + 8 * (lane & 1)) = make_float2(v0, v1);
        }
      }
    } else {
      // stmatrix x4: matrices (jj, rows r0), (jj, r0 + 8), (jj + 1, r0), (jj + 1, r0 + 8); lane gives a row of matrix lane / 8
      const int i = lane >> 3, r = 16 * warp + 8 * (i & 1) + (lane & 7);
      const uint32_t row_addr = smem_u32(sb) + r * 128;
#pragma unroll
      for (int jj = 0; jj < JPC; jj += 2) {
        const int j = c * JPC + jj;
        uint32_t p[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int jq = j + (q >> 1), h = q & 1;
          const float2 bq = b[jj + (q >> 1)];
          p[q] = pack_bf16x2(epi_act<EPI>(acc[4 * jq + 2 * h] + bq.x), epi_act<EPI>(acc[4 * jq + 2 * h + 1] + bq.y));
        }
        stmatrix_x4(row_addr + (((jj + (i >> 1)) ^ (r & 7)) << 4), p[0], p[1], p[2], p[3]);
      }
    }
    fence_proxy_async();   // this thread's smem writes -> visible to the async proxy (the TMA store)
    wg_bar_sync(bar);
    if (t == 0) {
      tma_store_2d(tma_out, sb, col0, row_wg);
      tma_store_commit();
    }
    buf ^= 1u;
  }
}

// dW += acc: the weight-gradient kernel's accumulate-into-gradient epilogue, straight from the accumulator fragment
// (rows r, r + 8; column pairs 8 j + 2 (lane % 4)) to global memory.  `row_w` = first row of this warp's 16-row slice.
template <int BN>
__device__ __forceinline__ void epilogue_accumulate(const float (&acc)[BN / 2], float* dw, int row_w, int n0, int M,
                                                    int N) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = n0 + 8 * j + 2 * (lane & 3);
    if (col >= N) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row_w + (lane >> 2) + 8 * h;
      if (row >= M) continue;
      float2* p = reinterpret_cast<float2*>(dw + (size_t)row * N + col);
      const float2 r = *p;
      *p = make_float2(acc[4 * j + 2 * h] + 0.f + r.x, acc[4 * j + 2 * h + 1] + 0.f + r.y);
    }
  }
}

// Barrier setup shared by both kernels: full[s] count 1 (+ tx), empty[s] one arrive per MMA warp of each CTA of the
// cluster that reads slot s.
template <int BN, int CL>
__device__ __forceinline__ void init_ring(const Ring<BN>& ring) {
  if (threadIdx.x == 0) {
    for (int s = 0; s < Cfg<BN>::STAGES; ++s) {
      mbar_init(&ring.full[s], 1);
      mbar_init(&ring.empty[s], 4 * NUM_MMA_WG * CL);
    }
    fence_barrier_init();
  }
}

// ===================================================================== main kernel
template <int BN, bool SK, int CL, int EPI>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_bf16_tc_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                    const __grid_constant__ CUtensorMap tma_out, EpiArgs ep, int M, int N, int K, SkArgs skargs) {
  using C = Cfg<BN>;
  constexpr int STAGES = C::STAGES;
  nerdev::pdl_launch_dependents();   // the next kernel of the stream may start its prologue while this one runs

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  if ((smem_u32(smem_raw) & 1023u) != 0u) __trap();  // SWIZZLE_128B tiles need 1024-B alignment
  const Ring<BN> ring(smem_raw);

  const int wg = threadIdx.x >> 7;
  const uint32_t rank = CL == 2 ? cluster_ctarank() : 0u;
  const int id = CL == 2 ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
  const int count = CL == 2 ? (int)(gridDim.x >> 1) : (int)gridDim.x;

  const int num_m = (M + CL * BM - 1) / (CL * BM);
  const int num_n = (N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_kb = (K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    tma_prefetch_desc(&tma_out);
  }
  init_ring<BN, CL>(ring);
  if constexpr (CL == 2) cluster_sync_all();  // barrier inits visible cluster-wide before any multicast / remote arrive
  else __syncthreads();
  // barriers and descriptor prefetch are set up: everything below touches global memory and must
  // wait for the previous kernel of the stream (no-op unless launched with the PDL attribute)
  nerdev::pdl_wait();

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x < 32 && elect_one()) {
      RingPos pos;
      SegIter it(SK, num_tiles, num_kb, id, count);
      int tile, kb0, kb1;
      while (it.next(tile, kb0, kb1)) {
        const int m_blk = tile / num_n, n_blk = tile - m_blk * num_n;
        const int row_a = (m_blk * CL + (int)rank) * BM;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&ring.empty[pos.stage], pos.phase ^ 1u);
          mbar_arrive_expect_tx(&ring.full[pos.stage], C::A_BYTES + C::B_BYTES);
          tma_load_2d(ring.a + pos.stage * C::A_BYTES, &tma_a, &ring.full[pos.stage], kb * BK, row_a);
          if constexpr (CL == 2)
            tma_load_2d_mc(ring.b + pos.stage * C::B_BYTES + rank * (C::B_BYTES / 2), &tma_b, &ring.full[pos.stage],
                           kb * BK, n_blk * BN + (int)rank * (BN / 2), (uint16_t)0x3);
          else
            tma_load_2d(ring.b + pos.stage * C::B_BYTES, &tma_b, &ring.full[pos.stage], kb * BK, n_blk * BN);
          pos.advance<STAGES>();
        }
      }
    }
  } else {
    // ===================== MMA + epilogue warpgroups =====================
    setmaxnreg_inc<232>();
    const int mw = wg - 1;                      // 64-row slice of the tile
    const int ctid = threadIdx.x - 128;         // 0 .. 255
    uint8_t* stage = ring.out + mw * 2 * OUT_CHUNK_BYTES;
    uint32_t buf = 0;
    uint32_t empty_peer[STAGES];
#pragma unroll
    for (int s = 0; s < STAGES; ++s) empty_peer[s] = CL == 2 ? mapa_u32(smem_u32(&ring.empty[s]), rank ^ 1u) : 0u;
    auto da = [](uint32_t addr, int k) { return make_wgmma_desc_sw128(addr + k * MMA_K * 2); };
    constexpr size_t SLOT = (size_t)BN * BM / 2;   // float2 per CTA slot
    float2* ws = reinterpret_cast<float2*>(skargs.ws);
    RingPos pos;
    SegIter it(SK, num_tiles, num_kb, id, count);
    int tile, kb0, kb1;
    float acc[BN / 2];
    while (it.next(tile, kb0, kb1)) {
      const int m_blk = tile / num_n, n_blk = tile - m_blk * num_n;
      const int row0 = (m_blk * CL + (int)rank) * BM;
      mma_kblocks<BN, STAGES, CL, 0, 0>(acc, ring, pos, kb0, kb1, (uint32_t)(mw * 64 * BK * 2), da, da, empty_peer);
      if (SK && kb0 > 0) {
        // contributor: park the raw partial accumulator of this CTA's first segment in its slot
        float2* p = ws + (size_t)blockIdx.x * SLOT + ctid;
#pragma unroll
        for (int i = 0; i < BN / 4; ++i) __stcg(p + (size_t)i * 256, make_float2(acc[2 * i], acc[2 * i + 1]));
        __threadfence();
        mma_bar_sync();
        if (ctid == 0) st_release_gpu(skargs.flags + blockIdx.x, 1);
        continue;
      }
      int c_first = 0, n_part = 0;
      if (SK && kb1 < num_kb) {
        // finisher: the following CTAs whose ranges start inside this tile hold its later k-blocks
        const long long U = (long long)num_tiles * num_kb, tile_end = (long long)(tile + 1) * num_kb;
        c_first = blockIdx.x + 1;
        for (int c = c_first; c < (int)gridDim.x; ++c) {
          const long long c0 = (long long)c * U / gridDim.x, c1 = (long long)(c + 1) * U / gridDim.x;
          if (c0 >= tile_end) break;
          if (c1 > c0) ++n_part; else if (n_part == 0) ++c_first;   // (empty ranges only occur when U < grid)
        }
        if (ctid == 0) {
          for (int c = 0; c < n_part; ++c) {
            unsigned spins = 0;
            while (ld_acquire_gpu(skargs.flags + c_first + c) == 0)
              if (++spins > (1u << 28)) __trap();   // never hang the GPU on a protocol bug
          }
        }
        mma_bar_sync();
        __threadfence();
        for (int c = 0; c < n_part; ++c) {
          const float2* p = ws + (size_t)(c_first + c) * SLOT + ctid;
#pragma unroll
          for (int i = 0; i < BN / 4; ++i) {
            const float2 v = __ldcg(p + (size_t)i * 256);
            acc[2 * i] += v.x;
            acc[2 * i + 1] += v.y;
          }
        }
      }
      if constexpr (EPI == NER_EPI_DIAG_DISCARD) {
        // diagnostic mode: store nothing, yet keep the accumulator live, or the compiler drops the wgmma of this
        // instantiation and the mode would time the loads only.  The smem write is under a condition no launch meets
        // (M >= 1 is checked on the host) but which the compiler cannot rule out.
        if (M < 0) {
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) reinterpret_cast<float*>(ring.a)[i * 256 + ctid] = acc[i];
        }
      } else {
        epilogue_tma<BN, EPI>(acc, ep, &tma_out, stage, buf, row0 + mw * 64, n_blk * BN, M, N);
      }
      if (n_part > 0) {
        mma_bar_sync();   // every MMA thread has consumed the parked partials
        if (ctid < 32)
          for (int c = ctid; c < n_part; c += 32) skargs.flags[c_first + c] = 0;
      }
    }
    if ((threadIdx.x & 127) == 0) tma_store_wait_all();   // staging stays valid until this warpgroup's stores are done
  }
  if constexpr (CL == 2) cluster_sync_all();  // no CTA leaves while its peer may still multicast into it / arrive on it
}

// ===================================================================== grouped weight gradients
// dW_p[k_in, n_out] += X_p^T[k_in, R] . dY_p[R, n_out]   for a group of problems p (the weight gradients of one encoder layer),
// ONE persistent launch: the tiles of all problems form one list (128 x 256 output tiles), so the 18..72 tiles of the single
// GEMMs (K = tokens: 50 k-blocks, a quarter to a half of the SMs idle per launch) become 216 per layer.
// Both operands are read AS THEY LIE in memory — X [R, k_in] and dY [R, n_out] are token-major, i.e. M / N contiguous and
// K (tokens) strided: "MN-major" (transposed) operands of wgmma.  A k-block is 64 tokens; the A tile arrives as two and the
// B tile as four {64 columns x 64 tokens} TMA boxes (SWIZZLE_128B), which is the canonical MN-major layout: 64-element
// blocks along M/N 8 KB apart (leading byte offset), 8-token groups 1 KB apart (stride byte offset); one MMA (K = 16) spans
// two token groups, consecutive MMAs advance the start address by 2 KB.  Each MMA warpgroup's 64 rows of A are one box.
// No bf16 transposes, no padded copies: TMA zero-fills the token rows past R.  Epilogue = fp32 accumulate-into-gradient (RES_F32).
constexpr int WG_MAXP = 6;
constexpr int WG_BN = 256;

struct WgradGroup {
  CUtensorMap a[WG_MAXP], b[WG_MAXP];
  float* dw[WG_MAXP];
  int m[WG_MAXP], n[WG_MAXP], b_col0[WG_MAXP];
  int tile_start[WG_MAXP + 1];
  int count, rows;
};

__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_wgrad_group_kernel(const __grid_constant__ WgradGroup grp) {
  constexpr int BN = WG_BN;
  using C = Cfg<BN>;
  constexpr int STAGES = C::STAGES;
  constexpr int BOX = 64 * 64 * 2;   // one {64 columns x 64 tokens} box
  nerdev::pdl_launch_dependents();

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  if ((smem_u32(smem_raw) & 1023u) != 0u) __trap();
  const Ring<BN> ring(smem_raw);

  const int wg = threadIdx.x >> 7;
  const int num_tiles = grp.tile_start[grp.count];
  const int num_kb = (grp.rows + BK - 1) / BK;

  init_ring<BN, 1>(ring);
  __syncthreads();
  nerdev::pdl_wait();

  auto locate = [&](int tile, int& p, int& m_blk, int& n_blk) {
    p = 0;
    while (p + 1 < grp.count && tile >= grp.tile_start[p + 1]) ++p;
    const int t = tile - grp.tile_start[p], num_n = grp.n[p] / BN;
    m_blk = t / num_n;
    n_blk = t - m_blk * num_n;
  };

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x < 32 && elect_one()) {
      RingPos pos;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int p, m_blk, n_blk;
        locate(tile, p, m_blk, n_blk);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&ring.empty[pos.stage], pos.phase ^ 1u);
          mbar_arrive_expect_tx(&ring.full[pos.stage], C::A_BYTES + C::B_BYTES);
#pragma unroll
          for (int i = 0; i < BM / 64; ++i)
            tma_load_2d(ring.a + pos.stage * C::A_BYTES + i * BOX, &grp.a[p], &ring.full[pos.stage], m_blk * BM + i * 64, kb * BK);
#pragma unroll
          for (int i = 0; i < BN / 64; ++i)
            tma_load_2d(ring.b + pos.stage * C::B_BYTES + i * BOX, &grp.b[p], &ring.full[pos.stage],
                        grp.b_col0[p] + n_blk * BN + i * 64, kb * BK);
          pos.advance<STAGES>();
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int mw = wg - 1;
    const int row_in_tile = mw * 64 + ((threadIdx.x >> 5) & 3) * 16;
    const uint32_t no_peer[STAGES] = {};
    auto da = [](uint32_t addr, int k) { return make_wgmma_desc_sw128(addr + k * 2048); };
    auto db = [](uint32_t addr, int k) { return make_wgmma_desc_sw128(addr + k * 2048, BOX); };
    RingPos pos;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int p, m_blk, n_blk;
      locate(tile, p, m_blk, n_blk);
      mma_kblocks<BN, STAGES, 1, 1, 1>(acc, ring, pos, 0, num_kb, (uint32_t)(mw * BOX), da, db, no_peer);
      epilogue_accumulate<BN>(acc, grp.dw[p], m_blk * BM + row_in_tile, n_blk * BN, grp.m[p], grp.n[p]);
    }
  }
}

// ===================================================================== FP8 (e4m3) GEMM with block scales
//   out[M,N] = epi( s_w[n] · Σ_j s_a[m,j] · (Σ_{k in block j} qa[m,k] · qw[n,k]) + bias[n] )
// A e4m3 [M,K] with fp32 scales s_a [M, K/128] (row m, columns [128j, 128j+128)); Wt e4m3 [N,K] with one fp32 scale per
// output channel s_w [N].  The persistent warp-specialised shape of gemm_bf16_tc_kernel with a 128 x 128 tile: a k-block is
// 128 e4m3 = 128 B, one SWIZZLE_128B row, so a ring stage holds as many bytes as the bf16 kernel's (Cfg<128>, Ring<128>).
// Per k-block four wgmma.m64n128k32 e4m3 accumulate into a temporary, which is then promoted into the fp32 accumulator with
// one FMA per element scaled by s_a[row, kb]: Hopper's FP8 wgmma accumulator keeps fewer mantissa bits than fp32, and
// promoting every 128 products bounds that loss to one block.  A warpgroup waits for its k-block's wgmma before promoting
// it (64 accumulator + 64 temporary registers per thread); the tensor cores stay fed by the other MMA warpgroup, whose
// wgmma runs while this one promotes.  Keeping a second k-block in flight through a second temporary makes ptxas serialise
// every wgmma (C7514: the promotion reads one accumulator while the other's group is pending) and spill.
// Epilogues: acc · s_w + bias -> bf16 through epilogue_tma, or GELU(acc · s_w + bias) -> e4m3 with 1 x 128 block scales.
constexpr int FP8_BN = 128;
constexpr int FP8_BK = 128;     // e4m3 per k-block = 128 B
constexpr int FP8_MMA_K = 32;

template <int EPI>
__host__ __device__ constexpr bool epi_e4m3() { return EPI == NER_EPI_GELU_TANH_E4M3 || EPI == NER_EPI_GELU_ERF_E4M3; }

// Four K = 32 wgmma of one k-block into the temporary `t` (the first one overwrites it), committed as one group.
__device__ __forceinline__ void fp8_issue(float (&t)[FP8_BN / 2], const Ring<FP8_BN>& ring, int stage, uint32_t a_off) {
  const uint32_t a_addr = smem_u32(ring.a + stage * Cfg<FP8_BN>::A_BYTES) + a_off;
  const uint32_t b_addr = smem_u32(ring.b + stage * Cfg<FP8_BN>::B_BYTES);
  reg_fence(t);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < FP8_BK / FP8_MMA_K; ++k)
    wgmma_m64n128k32_e4m3(t, make_wgmma_desc_sw128(a_addr + k * FP8_MMA_K), make_wgmma_desc_sw128(b_addr + k * FP8_MMA_K),
                          k > 0 ? 1u : 0u);
  wgmma_commit();
  reg_fence(t);
}

// acc += t · s_a of the fragment's rows (s0: row r, s1: row r + 8)
__device__ __forceinline__ void fp8_promote(float (&acc)[FP8_BN / 2], const float (&t)[FP8_BN / 2], float s0, float s1) {
#pragma unroll
  for (int i = 0; i < FP8_BN / 2; ++i) acc[i] = fmaf(t[i], (i & 2) ? s1 : s0, acc[i]);
}

// GELU(acc · s_w + bias) -> e4m3 with one scale per row and 128-column block.  A row's 128 tile columns sit in the four lanes
// of one quad, so the block amax is two shuffles.  The tanh form uses the accurate tanhf (not tanh.approx as the bf16
// epilogue does), so the quantised bytes are a function of the fp32 accumulator alone.  Values are quantised as x · (1/s)
// rather than x / s (the LayerNorm's form): the two differ by at most one fp32 ulp before the e4m3 rounding, and the 64
// divisions per thread were a measurable share of the FFN1 epilogue.  The warpgroup's 64 x 128 bytes are
// one 8 KB SWIZZLE_128B staging chunk, stored by TMA; the scales go straight to out_scale [M, N/128].
template <int EPI>
__device__ __forceinline__ void epilogue_e4m3(float (&acc)[FP8_BN / 2], const float* bias, float* out_scale,
                                              const CUtensorMap* tma_out, uint8_t* stage, uint32_t& buf, int row_wg, int n0,
                                              int M, int N) {
  const int t = threadIdx.x & 127, lane = t & 31, warp = t >> 5;
  const int bar = 1 + (threadIdx.x >> 7);
  const int r0 = 16 * warp + (lane >> 2);
  if (row_wg >= M) return;
  uint8_t* sb = stage + buf * OUT_CHUNK_BYTES;
  if (t == 0) tma_store_wait_read<1>();
  wg_bar_sync(bar);
  float amax[2] = {0.f, 0.f};
#pragma unroll
  for (int j = 0; j < FP8_BN / 8; ++j) {
    const int col = n0 + 8 * j + 2 * (lane & 3);
    const float2 b = bias != nullptr ? __ldg(reinterpret_cast<const float2*>(bias + col)) : make_float2(0.f, 0.f);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const float x = acc[4 * j + 2 * h + c] + (c ? b.y : b.x);
        float v;
        if constexpr (EPI == NER_EPI_GELU_ERF_E4M3) v = gelu_erf(x);
        else v = 0.5f * x * (1.f + tanhf(0.7978845608028654f * fmaf(0.044715f * x * x, x, x)));
        acc[4 * j + 2 * h + c] = v;
        amax[h] = fmaxf(amax[h], fabsf(v));
      }
    }
  }
  float inv[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    amax[h] = fmaxf(amax[h], __shfl_xor_sync(0xffffffffu, amax[h], 1));
    amax[h] = fmaxf(amax[h], __shfl_xor_sync(0xffffffffu, amax[h], 2));
    const float s = nerdev::e4m3_scale(amax[h]);
    inv[h] = __frcp_rn(s);
    const int row = row_wg + r0 + 8 * h;
    if ((lane & 3) == 0 && row < M) out_scale[(size_t)row * (N / FP8_BN) + n0 / FP8_BN] = s;
  }
#pragma unroll
  for (int j = 0; j < FP8_BN / 8; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r0 + 8 * h;
      const uint16_t q = nerdev::cvt_e4m3x2(acc[4 * j + 2 * h] * inv[h], acc[4 * j + 2 * h + 1] * inv[h]);
      *reinterpret_cast<uint16_t*>(sb + r * 128 + (((j >> 1) ^ (r & 7)) << 4) + 8 * (j & 1) + 2 * (lane & 3)) = q;
    }
  }
  fence_proxy_async();
  wg_bar_sync(bar);
  if (t == 0) {
    tma_store_2d(tma_out, sb, n0, row_wg);
    tma_store_commit();
  }
  buf ^= 1u;
}

template <int EPI>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_e4m3_tc_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                    const __grid_constant__ CUtensorMap tma_out, const float* __restrict__ a_scale,
                    const float* __restrict__ w_scale, const float* __restrict__ bias, float* __restrict__ out_scale, int M,
                    int N, int K) {
  using C = Cfg<FP8_BN>;
  constexpr int STAGES = C::STAGES;
  nerdev::pdl_launch_dependents();

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  if ((smem_u32(smem_raw) & 1023u) != 0u) __trap();
  const Ring<FP8_BN> ring(smem_raw);

  const int wg = threadIdx.x >> 7;
  const int num_n = N / FP8_BN;
  const int num_tiles = ((M + BM - 1) / BM) * num_n;
  const int num_kb = K / FP8_BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    tma_prefetch_desc(&tma_out);
  }
  init_ring<FP8_BN, 1>(ring);
  __syncthreads();
  nerdev::pdl_wait();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x < 32 && elect_one()) {
      RingPos pos;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / num_n, n_blk = tile - m_blk * num_n;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&ring.empty[pos.stage], pos.phase ^ 1u);
          mbar_arrive_expect_tx(&ring.full[pos.stage], C::A_BYTES + C::B_BYTES);
          tma_load_2d(ring.a + pos.stage * C::A_BYTES, &tma_a, &ring.full[pos.stage], kb * FP8_BK, m_blk * BM);
          tma_load_2d(ring.b + pos.stage * C::B_BYTES, &tma_b, &ring.full[pos.stage], kb * FP8_BK, n_blk * FP8_BN);
          pos.advance<STAGES>();
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int mw = wg - 1;
    const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
    uint8_t* stage = ring.out + mw * 2 * OUT_CHUNK_BYTES;
    uint32_t buf = 0;
    const uint32_t a_off = (uint32_t)(mw * 64 * FP8_BK);
    RingPos pos;
    float acc[FP8_BN / 2], tmp[FP8_BN / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_blk = tile / num_n, n_blk = tile - m_blk * num_n;
      const int row_wg = m_blk * BM + mw * 64, n0 = n_blk * FP8_BN;
      const int ra = row_wg + 16 * warp + (lane >> 2);
      // s_a rows of this thread's fragment (rows past M read row M - 1: TMA zero-fills their A, the value is unused)
      const float* sa0 = a_scale + (size_t)min(ra, M - 1) * num_kb;
      const float* sa1 = a_scale + (size_t)min(ra + 8, M - 1) * num_kb;
#pragma unroll
      for (int i = 0; i < FP8_BN / 2; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < num_kb; ++kb) {
        const float s0 = __ldg(sa0 + kb), s1 = __ldg(sa1 + kb);
        mbar_wait(&ring.full[pos.stage], pos.phase);
        fp8_issue(tmp, ring, pos.stage, a_off);
        wgmma_wait<0>();
        reg_fence(tmp);
        if (lane == 0) mbar_arrive(&ring.empty[pos.stage]);
        fp8_promote(acc, tmp, s0, s1);
        pos.advance<STAGES>();
      }
      // per-channel weight scale
#pragma unroll
      for (int j = 0; j < FP8_BN / 8; ++j) {
        const float2 sw = __ldg(reinterpret_cast<const float2*>(w_scale + n0 + 8 * j + 2 * (lane & 3)));
        acc[4 * j] *= sw.x;
        acc[4 * j + 1] *= sw.y;
        acc[4 * j + 2] *= sw.x;
        acc[4 * j + 3] *= sw.y;
      }
      if constexpr (epi_e4m3<EPI>())
        epilogue_e4m3<EPI>(acc, bias, out_scale, &tma_out, stage, buf, row_wg, n0, M, N);
      else
        epilogue_tma<FP8_BN, NER_EPI_BF16>(acc, EpiArgs{bias, nullptr}, &tma_out, stage, buf, row_wg, n0, M, N);
    }
    if ((threadIdx.x & 127) == 0) tma_store_wait_all();
  }
}

// ---------------------------------------------------------------- host side
// Row-major [rows, cols] of bf16 (f32 = false) or fp32 with a {box_cols, box_rows} box of 128-B rows, 128-byte swizzle.
int make_map_2d(CUtensorMap* map, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows, bool f32 = false) {
  EncodeTiledFn fn = tensor_map_encode_fn();
  if (fn == nullptr) return NER_ERR_NO_DRIVER;
  const uint32_t esz = f32 ? 4 : 2;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * esz};
  cuuint32_t box[2] = {128 / esz, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr),
                  dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? NER_OK : NER_ERR_INVALID_ARG;
}

// NER_GEMM_POLICY=1: "auto" picks the 128x256 tile whenever N allows instead of fitting waves (tuning hook).
int gemm_auto_policy() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("NER_GEMM_POLICY");
    v = e ? atoi(e) : 0;
  }
  return v;
}

int sm_count() { return ner_num_sms(); }

// Stream-K scratch: one slot of 128 x 256 fp32 per CTA + one flag per CTA, per (device, stream) so
// that GEMMs running concurrently on different streams never share slots.  Allocated on first use
// (the only memory this library owns), never freed, flags zeroed once (the kernel restores them).
struct SkScratch {
  int dev;
  cudaStream_t st;
  float4* ws;
  int* flags;
};
constexpr int kMaxSkScratch = 16;
SkScratch g_sk[kMaxSkScratch];
int g_sk_n = 0;
std::mutex g_sk_mu;

bool sk_scratch(cudaStream_t st, SkArgs* out) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return false;
  std::lock_guard<std::mutex> lk(g_sk_mu);
  for (int i = 0; i < g_sk_n; ++i)
    if (g_sk[i].dev == dev && g_sk[i].st == st) {
      out->ws = g_sk[i].ws;
      out->flags = g_sk[i].flags;
      return true;
    }
  if (g_sk_n == kMaxSkScratch) return false;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &cap) != cudaSuccess || cap != cudaStreamCaptureStatusNone) {
    (void)cudaGetLastError();
    return false;   // no allocation inside a graph capture: the caller falls back to whole-tile scheduling
  }
  const size_t slot = (size_t)(256 / 32) * 8 * 128 * sizeof(float4);
  float4* ws = nullptr;
  int* flags = nullptr;
  if (cudaMalloc(&ws, slot * sm_count()) != cudaSuccess) {
    (void)cudaGetLastError();
    return false;
  }
  if (cudaMalloc(&flags, sizeof(int) * sm_count()) != cudaSuccess || cudaMemset(flags, 0, sizeof(int) * sm_count()) != cudaSuccess) {
    (void)cudaGetLastError();
    cudaFree(ws);
    return false;
  }
  cudaDeviceSynchronize();
  g_sk[g_sk_n++] = SkScratch{dev, st, ws, flags};
  out->ws = ws;
  out->flags = flags;
  return true;
}

// Launch with PDL and, for CL = 2, clusters of two CTAs along x.
template <typename... KArgs, typename... Args>
cudaError_t launch_ex(void (*kern)(KArgs...), int grid, size_t smem, cudaStream_t st, int cl, Args... args) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(NUM_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  attr[1].id = cudaLaunchAttributeClusterDimension;
  attr[1].val.clusterDim.x = cl;
  attr[1].val.clusterDim.y = 1;
  attr[1].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 2;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

template <int BN, int CL, int EPI>
int launch_gemm(const void* A, const void* Wt, EpiArgs ep, void* out, int M, int N, int K, cudaStream_t st, bool sk) {
  CUtensorMap ma, mb, mo;
  int rc = make_map_2d(&ma, A, (uint64_t)M, (uint64_t)K, BM);
  if (rc != NER_OK) return rc;
  rc = make_map_2d(&mb, Wt, (uint64_t)N, (uint64_t)K, BN / CL);
  if (rc != NER_OK) return rc;
  rc = make_map_2d(&mo, out, (uint64_t)M, (uint64_t)N, 64, epi_f32<EPI>());   // one warpgroup's 64-row chunk
  if (rc != NER_OK) return rc;
  const size_t smem = Cfg<BN>::SMEM;
  const int tiles = ((M + CL * BM - 1) / (CL * BM)) * ((N + BN - 1) / BN);
  const int num_kb = (K + BK - 1) / BK;
  SkArgs ska{nullptr, nullptr};
  cudaError_t e;
  if constexpr (CL == 1) {
    // stream-K (128 x 128 / 128 x 256 tiles) needs every CTA co-resident (grid = #SMs) and at least one k-block unit per CTA
    if constexpr ((BN == 256 || BN == 128) && EPI != NER_EPI_DIAG_DISCARD) {
      if (sk && (long long)tiles * num_kb >= sm_count() && sk_scratch(st, &ska)) {
        e = launch_ex(gemm_bf16_tc_kernel<BN, true, 1, EPI>, sm_count(), smem, st, 1, ma, mb, mo, ep, M, N, K, ska);
        if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
        return ner_launch_status();
      }
    }
    e = launch_ex(gemm_bf16_tc_kernel<BN, false, 1, EPI>, tiles < sm_count() ? tiles : sm_count(), smem, st, 1, ma, mb, mo,
                  ep, M, N, K, ska);
  } else {
    const int max_pairs = sm_count() / 2;
    const int pairs = tiles < max_pairs ? tiles : max_pairs;
    e = launch_ex(gemm_bf16_tc_kernel<BN, false, 2, EPI>, 2 * pairs, smem, st, 2, ma, mb, mo, ep, M, N, K, ska);
  }
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  return ner_launch_status();
}

// The epilogue mode is a template parameter of the kernel: one instantiation per (tile, mode).
template <int BN, int CL>
int launch_gemm(const void* A, const void* Wt, EpiArgs ep, void* out, int M, int N, int K, int epilogue, cudaStream_t st,
                bool sk = false) {
  switch (epilogue) {
    case NER_EPI_F32: return launch_gemm<BN, CL, NER_EPI_F32>(A, Wt, ep, out, M, N, K, st, sk);
    case NER_EPI_BF16: return launch_gemm<BN, CL, NER_EPI_BF16>(A, Wt, ep, out, M, N, K, st, sk);
    case NER_EPI_GELU_TANH_BF16: return launch_gemm<BN, CL, NER_EPI_GELU_TANH_BF16>(A, Wt, ep, out, M, N, K, st, sk);
    case NER_EPI_GELU_ERF_BF16: return launch_gemm<BN, CL, NER_EPI_GELU_ERF_BF16>(A, Wt, ep, out, M, N, K, st, sk);
    case NER_EPI_RELU_BF16: return launch_gemm<BN, CL, NER_EPI_RELU_BF16>(A, Wt, ep, out, M, N, K, st, sk);
    case NER_EPI_RES_F32: return launch_gemm<BN, CL, NER_EPI_RES_F32>(A, Wt, ep, out, M, N, K, st, sk);
    case NER_EPI_RES_RELU_F32: return launch_gemm<BN, CL, NER_EPI_RES_RELU_F32>(A, Wt, ep, out, M, N, K, st, sk);
    case NER_EPI_DIAG_DISCARD: return launch_gemm<BN, CL, NER_EPI_DIAG_DISCARD>(A, Wt, ep, out, M, N, K, st, sk);
    default: return NER_ERR_INVALID_ARG;
  }
}

}  // namespace

// bf16 row-major [rows, cols] with a {64 columns, 64 rows} box, 128-byte swizzle (MN-major operand tiles).
static int make_map_bf16_box64(CUtensorMap* map, const void* ptr, uint64_t rows, uint64_t cols) {
  return make_map_2d(map, ptr, rows, cols, 64);
}

extern "C" int ner_wgrad_group_bf16(const ner_wgrad_problem* problems_host, int count, int rows, ner_stream_t stream) {
  if (count < 0 || rows < 0 || (count > 0 && !problems_host)) return NER_ERR_INVALID_ARG;
  if (count == 0 || rows == 0) return NER_OK;
  if (count > WG_MAXP) return NER_ERR_UNSUPPORTED;
  WgradGroup g;
  g.count = count;
  g.rows = rows;
  g.tile_start[0] = 0;
  for (int p = 0; p < count; ++p) {
    const ner_wgrad_problem& q = problems_host[p];
    if (!q.x_bf16 || !q.dy_bf16 || !q.dw || q.k_in < 1 || q.n_out < 1 || q.ld_x < q.k_in || q.dy_col0 < 0 ||
        q.ld_dy < q.dy_col0 + q.n_out)
      return NER_ERR_INVALID_ARG;
    if (q.k_in % BM != 0 || q.n_out % WG_BN != 0 || q.ld_x % 8 != 0 || q.ld_dy % 8 != 0 || q.dy_col0 % 64 != 0)
      return NER_ERR_UNSUPPORTED;
    if ((reinterpret_cast<uintptr_t>(q.x_bf16) & 15) || (reinterpret_cast<uintptr_t>(q.dy_bf16) & 15) ||
        (reinterpret_cast<uintptr_t>(q.dw) & 15))
      return NER_ERR_INVALID_ARG;
    int rc = make_map_bf16_box64(&g.a[p], q.x_bf16, (uint64_t)rows, (uint64_t)q.ld_x);
    if (rc != NER_OK) return rc;
    rc = make_map_bf16_box64(&g.b[p], q.dy_bf16, (uint64_t)rows, (uint64_t)q.ld_dy);
    if (rc != NER_OK) return rc;
    g.dw[p] = q.dw;
    g.m[p] = q.k_in;
    g.n[p] = q.n_out;
    g.b_col0[p] = q.dy_col0;
    g.tile_start[p + 1] = g.tile_start[p] + (q.k_in / BM) * (q.n_out / WG_BN);
  }
  for (int p = count; p < WG_MAXP; ++p) {
    g.a[p] = g.a[0]; g.b[p] = g.b[0];
    g.dw[p] = nullptr; g.m[p] = g.n[p] = g.b_col0[p] = 0;
    g.tile_start[p + 1] = g.tile_start[count];
  }
  const int tiles = g.tile_start[count];
  const int grid = tiles < sm_count() ? tiles : sm_count();
  cudaError_t e = launch_ex(gemm_wgrad_group_kernel, grid, Cfg<WG_BN>::SMEM, static_cast<cudaStream_t>(stream), 1, g);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  return ner_launch_status();
}

extern "C" int ner_gemm_bf16(const void* A, const void* Wt, const float* bias, const float* residual, void* out,
                             int M, int N, int K, int epilogue, int tile_n, ner_stream_t stream) {
  if (M < 0 || N < 1 || K < 1) return NER_ERR_INVALID_ARG;
  if (M == 0) return NER_OK;
  if (!A || !Wt || !out) return NER_ERR_INVALID_ARG;
  if ((epilogue < NER_EPI_F32 || epilogue > NER_EPI_RES_RELU_F32) && epilogue != NER_EPI_DIAG_DISCARD) return NER_ERR_INVALID_ARG;
  if ((epilogue == NER_EPI_RES_F32 || epilogue == NER_EPI_RES_RELU_F32) && !residual) return NER_ERR_INVALID_ARG;
  if ((K % 8) != 0 || (N % 32) != 0) return NER_ERR_UNSUPPORTED;  // 16-B TMA strides, 32-col epilogue chunks
  if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(Wt) & 15) ||
      (reinterpret_cast<uintptr_t>(out) & 15))
    return NER_ERR_INVALID_ARG;
  // the epilogue reads bias and residual as float2 column pairs
  if ((reinterpret_cast<uintptr_t>(bias) & 7) || (reinterpret_cast<uintptr_t>(residual) & 7)) return NER_ERR_INVALID_ARG;
  EpiArgs ep{bias, residual};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int bn = tile_n;
  bool sk = false;
  if (bn == NER_TILE_SK_256 || bn == NER_TILE_SK_128) {
    sk = true;
    bn = (bn == NER_TILE_SK_256) ? 256 : 128;
  } else if (bn == NER_TILE_AUTO_THROUGHPUT || (bn == 0 && gemm_auto_policy() == 1)) {
    // throughput policy: several streams keep the SMs busy, so take the tile with the best FLOP rate
    bn = (N % 256 == 0) ? 256 : (N % 192 == 0) ? 192 : 128;
  }
  if (bn == 0) {
    // Cost model in units of one 128x256 k-block per CTA.  Whole-tile scheduling: ceil(tiles/SMs) waves
    // of num_kb k-blocks times the relative k-block cost of the tile width (narrower tiles re-read the A
    // tile more often per FLOP).  Stream-K (128x256 tiles): every CTA gets ceil(tiles*num_kb/SMs) k-blocks
    // plus a fixed charge for parking / adding one partial accumulator.  Re-checked on an H100 SXM (400 W limit) with the
    // TMA-store epilogue over the encoder shapes at 3549 and 12202 rows (scripts/bench_kernels.py gemm): it picks the
    // fastest of 128 / 192 / 256 within 3 % (the run-to-run spread) in all ten, and stream-K, 15-72 % slower there, is
    // never chosen.
    const int mt = (M + BM - 1) / BM, sms = sm_count(), num_kb = (K + BK - 1) / BK;
    const int cand[3] = {256, 192, 128};
    const float cost[3] = {1.00f, 0.80f, 0.64f};
    float best = 1e30f;
    bn = 128;
    for (int i = 0; i < 3; ++i) {
      if (N % cand[i] != 0) continue;
      const int tiles = mt * (N / cand[i]);
      const float t = (float)((tiles + sms - 1) / sms) * cost[i] * (float)num_kb;
      if (t < best - 1e-6f) {
        best = t;
        bn = cand[i];
      }
    }
    if (N % 256 == 0) {
      const long long units = (long long)mt * (N / 256) * num_kb;
      const float t_sk = (float)((units + sms - 1) / sms) + kSkFixupCost;
      if (units >= sms && t_sk < 0.9f * best) {
        sk = true;
        bn = 256;
      }
    }
  }
  switch (bn) {
    case 256: return launch_gemm<256, 1>(A, Wt, ep, out, M, N, K, epilogue, st, sk);
    case 192: return launch_gemm<192, 1>(A, Wt, ep, out, M, N, K, epilogue, st);
    case 128: return launch_gemm<128, 1>(A, Wt, ep, out, M, N, K, epilogue, st, sk);
    case 64: return launch_gemm<64, 1>(A, Wt, ep, out, M, N, K, epilogue, st);
    case NER_TILE_2CTA_256: return launch_gemm<256, 2>(A, Wt, ep, out, M, N, K, epilogue, st);
    case NER_TILE_2CTA_128: return launch_gemm<128, 2>(A, Wt, ep, out, M, N, K, epilogue, st);
    default: return NER_ERR_INVALID_ARG;
  }
}

namespace {
// e4m3 row-major [rows, cols] (one byte per element) with a {128 columns, box_rows} box, 128-byte swizzle.
int make_map_e4m3(CUtensorMap* map, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  EncodeTiledFn fn = tensor_map_encode_fn();
  if (fn == nullptr) return NER_ERR_NO_DRIVER;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols};
  cuuint32_t box[2] = {128, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? NER_OK : NER_ERR_INVALID_ARG;
}

template <int EPI>
int launch_gemm_e4m3(const void* A, const float* a_scale, const void* Wt, const float* w_scale, const float* bias, void* out,
                     float* out_scale, int M, int N, int K, cudaStream_t st) {
  CUtensorMap ma, mb, mo;
  int rc = make_map_e4m3(&ma, A, (uint64_t)M, (uint64_t)K, BM);
  if (rc != NER_OK) return rc;
  rc = make_map_e4m3(&mb, Wt, (uint64_t)N, (uint64_t)K, FP8_BN);
  if (rc != NER_OK) return rc;
  rc = epi_e4m3<EPI>() ? make_map_e4m3(&mo, out, (uint64_t)M, (uint64_t)N, 64) : make_map_2d(&mo, out, (uint64_t)M, (uint64_t)N, 64);
  if (rc != NER_OK) return rc;
  const int tiles = ((M + BM - 1) / BM) * (N / FP8_BN);
  const cudaError_t e = launch_ex(gemm_e4m3_tc_kernel<EPI>, tiles < sm_count() ? tiles : sm_count(), Cfg<FP8_BN>::SMEM, st, 1,
                                  ma, mb, mo, a_scale, w_scale, bias, out_scale, M, N, K);
  if (e != cudaSuccess) return NER_ERR_CUDA_BASE - (int)e;
  return ner_launch_status();
}
}  // namespace

extern "C" int ner_gemm_e4m3(const void* A, const float* a_scale, const void* Wt, const float* w_scale, const float* bias,
                             void* out, float* out_scale, int M, int N, int K, int epilogue, ner_stream_t stream) {
  if (M < 0 || N < 1 || K < 1) return NER_ERR_INVALID_ARG;
  if (epilogue != NER_EPI_BF16 && epilogue != NER_EPI_GELU_TANH_E4M3 && epilogue != NER_EPI_GELU_ERF_E4M3)
    return NER_ERR_INVALID_ARG;
  if (K % FP8_BK != 0 || N % FP8_BN != 0) return NER_ERR_UNSUPPORTED;   // whole 128-wide scale blocks and tiles
  if (M == 0) return NER_OK;
  const bool q_out = epilogue != NER_EPI_BF16;
  if (!A || !a_scale || !Wt || !w_scale || !out || (q_out && !out_scale)) return NER_ERR_INVALID_ARG;
  if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(Wt) & 15) || (reinterpret_cast<uintptr_t>(out) & 15))
    return NER_ERR_INVALID_ARG;
  // w_scale and bias are read as float2 column pairs
  if ((reinterpret_cast<uintptr_t>(w_scale) & 7) || (reinterpret_cast<uintptr_t>(bias) & 7)) return NER_ERR_INVALID_ARG;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (epilogue) {
    case NER_EPI_BF16: return launch_gemm_e4m3<NER_EPI_BF16>(A, a_scale, Wt, w_scale, bias, out, out_scale, M, N, K, st);
    case NER_EPI_GELU_TANH_E4M3:
      return launch_gemm_e4m3<NER_EPI_GELU_TANH_E4M3>(A, a_scale, Wt, w_scale, bias, out, out_scale, M, N, K, st);
    default: return launch_gemm_e4m3<NER_EPI_GELU_ERF_E4M3>(A, a_scale, Wt, w_scale, bias, out, out_scale, M, N, K, st);
  }
}
