// K-gemm: persistent, warp-specialised bf16 GEMM on the Hopper tensor cores (wgmma) for every dense contraction of the
// SOME conformer (reference call sites: Gconform.py:29-34 conform_ffn, base_attention.py:31-32,46 to_q/to_kv/to_out,
// base_conv.py:65,69 pointwise convs, Gconform.py:85-87 glu1/glu2, Gconform.py:124-125,135-136 inln/inln1/outln).
//
//   C[M, N] = epilogue(A[M, K] . W[N, K]^T)        A, W bf16 row-major (both K-major), fp32 accumulate
//
// Roles (384 threads = 3 warpgroups, 1 CTA / SM, grid = #SMs, static round-robin schedule over 128 x 256 tiles, N fastest):
//   warpgroup 0     TMA producer (one thread): A box 128x64 + W box 256x64 (128-B swizzle) into a 4-stage smem ring;
//                   gives its registers to the consumers (setmaxnreg)
//   warpgroups 1-2  consumers: rows [64 c, 64 c + 64) of the tile, wgmma m64n256k16 from shared memory into 128 fp32
//                   registers per thread, one k-block in flight while the previous one's stage is released; then the fused
//                   epilogue (bias / SiLU / GLU / residual / LayerNorm fold / sigmoid / softmax) straight from the
//                   accumulator registers: each quad of lanes stores 8 consecutive columns of a row (32 B in fp32, 16 B in bf16).
// Up to two independent problems (the "midi" and "bound" streams: same shapes, different weights) run in one launch
// (groups = 2).
#include "host_common.h"
#include "sm90_ptx.cuh"

#include <string.h>

#include "../../include/some_b200.h"

namespace some {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = 256;
constexpr int BLOCK_K = 64;
constexpr int WGMMA_K = 16;
constexpr int STAGES = 4;
constexpr int GEMM_THREADS = 384;
constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;   // 16 KB
constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;   // 32 KB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int GEMM_SMEM = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
static_assert(GEMM_SMEM <= 232448, "gemm_kernel: shared memory over the 227 KB per-CTA limit");
constexpr int ACC = BLOCK_N / 2;   // accumulator registers per consumer thread

struct GemmGroup {
  const float* bias;   // [N] in packed-column order, or nullptr
  void* out;           // bf16 or f32, row pitch ld_out elements
  const float* resid;  // f32 [M, ld_out] or nullptr (may alias out)
  const float* ln_s;   // LayerNorm-folded consumers: column sums of W' [N]
  float* ln_stats;     // f32 [M][SOME_LN_SLOTS][2] partial (sum x, sum x^2): written by producers, read by consumers
  __nv_bfloat16* out_bf16;   // LayerNorm producers: bf16 copy of out, row pitch ld_out
};

struct GemmParams {
  int M, N, K;
  int groups;
  int ld_out;
  int n_valid;  // softmax / sigmoid heads: number of real columns
  int ln_parts; // LayerNorm-folded consumers: valid slots per row of ln_stats
  float alpha;
  GemmGroup g[2];
};

template <int EPI>
struct EpiCfg {
  static constexpr bool LNP = EPI == SOME_EPI_RESID_F32_LN || EPI == SOME_EPI_GLU_RESID_F32_LN;
  static constexpr bool LNC = EPI == SOME_EPI_LN_STORE_BF16 || EPI == SOME_EPI_LN_SILU_BF16 || EPI == SOME_EPI_LN_GLU_BF16;
  // the LayerNorm variants share the store path of their plain epilogue
  static constexpr int BASE = LNC ? EPI - SOME_EPI_LN_STORE_BF16
                              : EPI == SOME_EPI_RESID_F32_LN ? SOME_EPI_RESID_F32
                              : EPI == SOME_EPI_GLU_RESID_F32_LN ? SOME_EPI_GLU_RESID_F32 : EPI;
};

// Row statistics of the LayerNorm input from the producers' partial sums (nn.LayerNorm: biased variance, eps 1e-5).
__device__ __forceinline__ void ln_row_coeffs(const GemmParams& p, const GemmGroup& g, int row, float& ra, float& nmu) {
  float s = 0.f, q = 0.f;
  if (row < p.M) {
    const float2* st = reinterpret_cast<const float2*>(g.ln_stats) + (size_t)row * SOME_LN_SLOTS;
    for (int i = 0; i < p.ln_parts; ++i) {
      const float2 t = st[i];
      s += t.x, q += t.y;
    }
  }
  const float inv_d = 1.0f / static_cast<float>(p.K);
  const float mean = s * inv_d;
  const float var = fmaxf(fmaf(-mean, mean, q * inv_d), 0.f);
  ra = rsqrtf(var + 1e-5f);
  nmu = -mean;
}

__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}

// Epilogue of one consumer thread: acc holds rows row0 and row0 + 8, columns col_tile + 8 j + 2 q + {0, 1} (j < 32).
// GLU: packed columns come in 32-column groups [16 "out" | 16 "gate"], so the gate of acc[4 j + i] is acc[4 (j + 2) + i]
// (j % 4 < 2) and output channel (col_tile + 32 G) / 2 + 8 jj + 2 q + e belongs to group G, j = 4 G + jj.
// LayerNorm producers: slot col / 128 of ln_stats gets (sum x, sum x^2) of the row over those 128 accumulator columns.
template <int EPI>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, const GemmGroup& g, float (&acc)[ACC], int row0,
                                              int col_tile, int q) {
  using Cfg = EpiCfg<EPI>;
  constexpr int BASE = Cfg::BASE;
  const int rows[2] = {row0, row0 + 8};
  const bool row_ok[2] = {rows[0] < p.M, rows[1] < p.M};

  // ---- bias, or the folded LayerNorm:  LN(x) . W^T + bias = rstd * (acc - mean * s_n) + bias'_n  (s_n = ln_s, bias' = bias)
  [[maybe_unused]] float ra[2] = {1.f, 1.f}, nmu[2] = {0.f, 0.f};
  if constexpr (Cfg::LNC) {
    ln_row_coeffs(p, g, rows[0], ra[0], nmu[0]);
    ln_row_coeffs(p, g, rows[1], ra[1], nmu[1]);
  }
  if (Cfg::LNC || g.bias != nullptr) {
#pragma unroll
    for (int j = 0; j < ACC / 4; ++j) {
      const int col = col_tile + 8 * j + 2 * q;
      if (col >= p.N) continue;   // ragged head tile: bias arrays are padded to 32 floats, not to the tile
      const float2 b = __ldg(reinterpret_cast<const float2*>(g.bias + col));
      if constexpr (Cfg::LNC) {
        const float2 sn = __ldg(reinterpret_cast<const float2*>(g.ln_s + col));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          acc[4 * j + 2 * h] = fmaf(fmaf(sn.x, nmu[h], acc[4 * j + 2 * h]), ra[h], b.x);
          acc[4 * j + 2 * h + 1] = fmaf(fmaf(sn.y, nmu[h], acc[4 * j + 2 * h + 1]), ra[h], b.y);
        }
      } else {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          acc[4 * j + 2 * h] += b.x;
          acc[4 * j + 2 * h + 1] += b.y;
        }
      }
    }
  }

  if constexpr (BASE == SOME_EPI_STORE_BF16 || BASE == SOME_EPI_SILU_BF16) {
#pragma unroll
    for (int j = 0; j < ACC / 4; ++j) {
      const int col = col_tile + 8 * j + 2 * q;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if constexpr (BASE == SOME_EPI_SILU_BF16) v0 = silu_fast(v0), v1 = silu_fast(v1);
        if (row_ok[h])
          *reinterpret_cast<uint32_t*>(static_cast<__nv_bfloat16*>(g.out) + (size_t)rows[h] * p.ld_out + col) = pack_bf16x2(v0, v1);
      }
    }
  } else if constexpr (BASE == SOME_EPI_GLU_BF16) {
#pragma unroll
    for (int G = 0; G < ACC / 16; ++G) {
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        const int j = 4 * G + jj;
        const int oc = (col_tile >> 1) + 16 * G + 8 * jj + 2 * q;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float o0 = acc[4 * j + 2 * h] * sigmoid_fast(acc[4 * (j + 2) + 2 * h]);
          const float o1 = acc[4 * j + 2 * h + 1] * sigmoid_fast(acc[4 * (j + 2) + 2 * h + 1]);
          if (row_ok[h])
            *reinterpret_cast<uint32_t*>(static_cast<__nv_bfloat16*>(g.out) + (size_t)rows[h] * p.ld_out + oc) = pack_bf16x2(o0, o1);
        }
      }
    }
  } else if constexpr (BASE == SOME_EPI_RESID_F32 || BASE == SOME_EPI_GLU_RESID_F32) {
    constexpr bool GLU = BASE == SOME_EPI_GLU_RESID_F32;
    [[maybe_unused]] float st_s[2][2] = {}, st_q[2][2] = {};   // [row half][128-column slot of the tile]
#pragma unroll
    for (int j = 0; j < ACC / 4; ++j) {
      if (GLU && (j & 3) >= 2) continue;   // gate columns: consumed with their "out" partners
      const int oc = GLU ? (col_tile >> 1) + 16 * (j >> 2) + 8 * (j & 3) + 2 * q : col_tile + 8 * j + 2 * q;
      const int slot = j >> 4;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if constexpr (GLU) {
          v0 *= sigmoid_fast(acc[4 * (j + 2) + 2 * h]);
          v1 *= sigmoid_fast(acc[4 * (j + 2) + 2 * h + 1]);
        }
        if (row_ok[h]) {
          const size_t off = (size_t)rows[h] * p.ld_out + oc;
          const float2 r = *reinterpret_cast<const float2*>(g.resid + off);
          float2 x;
          if constexpr (GLU) x = make_float2(r.x + v0, r.y + v1);
          else x = make_float2(fmaf(v0, p.alpha, r.x), fmaf(v1, p.alpha, r.y));   // alpha * (acc + bias) + resid
          *reinterpret_cast<float2*>(static_cast<float*>(g.out) + off) = x;
          if constexpr (Cfg::LNP) {
            st_s[h][slot] += x.x + x.y;
            st_q[h][slot] = fmaf(x.x, x.x, fmaf(x.y, x.y, st_q[h][slot]));
            *reinterpret_cast<uint32_t*>(g.out_bf16 + off) = pack_bf16x2(x.x, x.y);
          }
        }
      }
    }
    if constexpr (Cfg::LNP) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int sl = 0; sl < 2; ++sl) {
          const float s = quad_sum(st_s[h][sl]), qq = quad_sum(st_q[h][sl]);
          if (q == 0 && row_ok[h])
            reinterpret_cast<float2*>(g.ln_stats)[(size_t)rows[h] * SOME_LN_SLOTS + (col_tile >> 7) + sl] = make_float2(s, qq);
        }
      }
    }
  } else if constexpr (BASE == SOME_EPI_BIAS_F32 || BASE == SOME_EPI_SIGMOID_F32) {
#pragma unroll
    for (int j = 0; j < ACC / 4; ++j) {
      const int col = col_tile + 8 * j + 2 * q;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float v = acc[4 * j + 2 * h + e];
          if constexpr (BASE == SOME_EPI_SIGMOID_F32) v = 1.0f / (1.0f + __expf(-v));
          if (row_ok[h] && col + e < p.n_valid) static_cast<float*>(g.out)[(size_t)rows[h] * p.ld_out + col + e] = v;
        }
      }
    }
  } else {
    static_assert(BASE == SOME_EPI_SOFTMAX_F32, "unknown epilogue");
    // the whole row is in this tile (N <= 256): a quad of lanes holds it
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < ACC / 4; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (8 * j + 2 * q + e < p.n_valid) mx = fmaxf(mx, acc[4 * j + 2 * h + e]);
      mx = quad_max(mx);
      float sum = 0.f;   // exponentials in place: the row is read once more only to be scaled and stored
#pragma unroll
      for (int j = 0; j < ACC / 4; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& v = acc[4 * j + 2 * h + e];
          v = 8 * j + 2 * q + e < p.n_valid ? __expf(v - mx) : 0.f;
          sum += v;
        }
      const float inv = 1.0f / quad_sum(sum);
      if (row_ok[h]) {
        float* dst = static_cast<float*>(g.out) + (size_t)rows[h] * p.ld_out;
#pragma unroll
        for (int j = 0; j < ACC / 4; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * j + 2 * q + e;
            if (col < p.n_valid) dst[col] = acc[4 * j + 2 * h + e] * inv;
          }
      }
    }
  }
}

template <int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmB0,
            const __grid_constant__ CUtensorMap tmA1, const __grid_constant__ CUtensorMap tmB1, const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);   // [STAGES]
  uint64_t* empty_bar = full_bar + STAGES;                                          // [STAGES]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  const int num_m = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int num_n = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int tiles_per_group = num_m * num_n;
  const int num_tiles = tiles_per_group * p.groups;
  const int num_kb = (p.K + BLOCK_K - 1) / BLOCK_K;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA0);
    tma_prefetch_desc(&tmB0);
    if (p.groups > 1) {
      tma_prefetch_desc(&tmA1);
      tma_prefetch_desc(&tmB1);
    }
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);   // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  griddep_launch();     // programmatic dependent launch: the next kernel may start its own prologue ...
  griddep_wait();       // ... and this one touches activations only after its predecessor has completed

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one_sync()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int grp = tile / tiles_per_group;
        const int t = tile - grp * tiles_per_group;
        const int m_blk = t / num_n, n_blk = t - m_blk * num_n;
        const CUtensorMap* ta = grp == 0 ? &tmA0 : &tmA1;
        const CUtensorMap* tb = grp == 0 ? &tmB0 : &tmB1;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);   // out-of-bounds rows are zero-filled and still counted
          uint8_t* sa = smem + stage * STAGE_BYTES;
          tma_load_2d(sa, ta, &full_bar[stage], kb * BLOCK_K, m_blk * BLOCK_M);
          tma_load_2d(sa + A_BYTES, tb, &full_bar[stage], kb * BLOCK_K, n_blk * BLOCK_N);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    __syncwarp();
  } else {
    setmaxnreg_inc<232>();
    const int cw = wg - 1;   // consumer warpgroup: rows [64 cw, 64 cw + 64) of the tile
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int grp = tile / tiles_per_group;
      const int t = tile - grp * tiles_per_group;
      const int m_blk = t / num_n, n_blk = t - m_blk * num_n;
      float acc[ACC];
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
        const uint64_t adesc = gmma_desc_kmajor_sw128(sa + cw * 64 * 128);
        const uint64_t bdesc = gmma_desc_kmajor_sw128(sa + A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WGMMA_K; ++k)   // +16 bf16 = 32 B along K inside the 128-B swizzle atom: +2 in (addr >> 4)
          wgmma_m64n256k16_ss(acc, adesc + 2 * k, bdesc + 2 * k, (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();   // the previous k-block's MMAs have finished reading their stage
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_reg_fence(acc);
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
      const GemmGroup g = grp == 0 ? p.g[0] : p.g[1];   // no dynamic index into the parameter space (a local copy)
      epilogue_tile<EPI>(p, g, acc, m_blk * BLOCK_M + cw * 64 + (warp & 3) * 16 + (lane >> 2), n_blk * BLOCK_N,
                         lane & 3);
    }
  }
}

template <int EPI>
static int launch_gemm(const CUtensorMap* maps, const GemmParams& p, cudaStream_t stream) {
  auto kern = gemm_kernel<EPI>;
  static bool configured[kMaxDevices] = {};   // function attributes are per device
  const int dev_ = device_index();
  if (!configured[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM);
    SOME_REQUIRE(e == cudaSuccess, "cudaFuncSetAttribute(gemm, %d B smem): %s", GEMM_SMEM, cudaGetErrorString(e));
    configured[dev_] = true;
  }
  const int num_m = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int num_n = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int tiles = num_m * num_n * p.groups;
  int grid = num_sms();
  if (tiles < grid) grid = tiles;
  launch_pdl(kern, dim3(grid), dim3(GEMM_THREADS), GEMM_SMEM, stream, maps[0], maps[1], maps[2], maps[3], p);
  return check_launch("some_gemm");
}

}  // namespace some

using namespace some;

extern "C" int some_gemm(const some_gemm_args* a, cudaStream_t stream) {
  SOME_REQUIRE(a != nullptr, "some_gemm: null args");
  SOME_REQUIRE(a->groups == 1 || a->groups == 2, "some_gemm: groups must be 1 or 2 (got %d)", a->groups);
  SOME_REQUIRE(a->M >= 0 && a->N > 0 && a->K > 0, "some_gemm: bad shape M=%d N=%d K=%d", a->M, a->N, a->K);
  if (a->M == 0) return 0;
  SOME_REQUIRE(a->K % 8 == 0, "some_gemm: K must be a multiple of 8 (16-byte TMA pitch), got %d", a->K);
  const int epi = a->epilogue;
  const bool head = (epi == SOME_EPI_SOFTMAX_F32 || epi == SOME_EPI_SIGMOID_F32 || epi == SOME_EPI_BIAS_F32);
  if (!head) SOME_REQUIRE(a->N % 256 == 0, "some_gemm: N must be a multiple of 256 for epilogue %d (got %d)", epi, a->N);
  if (epi == SOME_EPI_SOFTMAX_F32) SOME_REQUIRE(a->N <= 256, "some_gemm: softmax epilogue needs N <= 256");
  const bool ln_consumer = epi == SOME_EPI_LN_STORE_BF16 || epi == SOME_EPI_LN_SILU_BF16 || epi == SOME_EPI_LN_GLU_BF16;
  const bool ln_producer = epi == SOME_EPI_RESID_F32_LN || epi == SOME_EPI_GLU_RESID_F32_LN;
  const bool glu_resid = epi == SOME_EPI_GLU_RESID_F32 || epi == SOME_EPI_GLU_RESID_F32_LN;
  const bool needs_resid = epi == SOME_EPI_RESID_F32 || epi == SOME_EPI_RESID_F32_LN || glu_resid;
  GemmParams p;
  p.M = a->M;
  p.N = a->N;
  p.K = a->K;
  p.groups = a->groups;
  p.ld_out = a->ld_out;
  p.n_valid = a->N;
  p.alpha = a->alpha;
  p.ln_parts = a->ln_parts;
  if (ln_consumer)
    SOME_REQUIRE(a->ln_parts >= 1 && a->ln_parts <= SOME_LN_SLOTS, "some_gemm: ln_parts must be in [1, %d] (got %d)",
                 SOME_LN_SLOTS, a->ln_parts);
  // one slot per 128 accumulator columns (= 128 outputs, or 64 after a GLU)
  if (ln_producer)
    SOME_REQUIRE(a->N / 128 <= SOME_LN_SLOTS, "some_gemm: LayerNorm producer output too wide (N=%d)", a->N);
  CUtensorMap maps[4];
  for (int g = 0; g < 2; ++g) {
    const int s = g < a->groups ? g : 0;
    SOME_REQUIRE(a->A[s] != nullptr && a->W[s] != nullptr && a->out[s] != nullptr, "some_gemm: null pointer in group %d", s);
    if (make_tmap_bf16_2d(&maps[2 * g], a->A[s], a->M, a->K, a->lda, BLOCK_M)) return -1;
    if (make_tmap_bf16_2d(&maps[2 * g + 1], a->W[s], a->N, a->K, a->K, BLOCK_N)) return -1;
    p.g[g].bias = a->bias[s];
    p.g[g].out = a->out[s];
    p.g[g].resid = a->resid[s];
    p.g[g].ln_s = a->ln_s[s];
    p.g[g].ln_stats = a->ln_stats[s];
    p.g[g].out_bf16 = reinterpret_cast<__nv_bfloat16*>(a->out_bf16[s]);
    if (needs_resid) {
      const int out_cols = glu_resid ? a->N / 2 : a->N;
      SOME_REQUIRE(a->resid[s] != nullptr, "some_gemm: epilogue %d needs a residual pointer (group %d)", epi, s);
      SOME_REQUIRE(a->ld_out % 4 == 0 && out_cols <= a->ld_out, "some_gemm: bad ld_out %d for %d output columns", a->ld_out, out_cols);
      if (ln_producer)
        SOME_REQUIRE(a->out_bf16[s] != nullptr && a->ln_stats[s] != nullptr,
                     "some_gemm: LayerNorm producer epilogue %d needs out_bf16 and ln_stats (group %d)", epi, s);
    }
    if (!head && !needs_resid) {   // bf16 epilogues: bf16 pairs stored as 32-bit words
      const int out_cols = (epi == SOME_EPI_GLU_BF16 || epi == SOME_EPI_LN_GLU_BF16) ? a->N / 2 : a->N;
      SOME_REQUIRE(a->ld_out % 8 == 0 && out_cols <= a->ld_out, "some_gemm: bad ld_out %d for %d bf16 output columns", a->ld_out, out_cols);
    }
    if (ln_consumer)
      SOME_REQUIRE(a->ln_s[s] != nullptr && a->ln_stats[s] != nullptr && a->bias[s] != nullptr,
                   "some_gemm: LayerNorm consumer epilogue %d needs bias, ln_s and ln_stats (group %d)", epi, s);
  }
  switch (epi) {
    case SOME_EPI_STORE_BF16: return launch_gemm<SOME_EPI_STORE_BF16>(maps, p, stream);
    case SOME_EPI_SILU_BF16: return launch_gemm<SOME_EPI_SILU_BF16>(maps, p, stream);
    case SOME_EPI_GLU_BF16: return launch_gemm<SOME_EPI_GLU_BF16>(maps, p, stream);
    case SOME_EPI_RESID_F32: return launch_gemm<SOME_EPI_RESID_F32>(maps, p, stream);
    case SOME_EPI_GLU_RESID_F32: return launch_gemm<SOME_EPI_GLU_RESID_F32>(maps, p, stream);
    case SOME_EPI_LN_STORE_BF16: return launch_gemm<SOME_EPI_LN_STORE_BF16>(maps, p, stream);
    case SOME_EPI_LN_SILU_BF16: return launch_gemm<SOME_EPI_LN_SILU_BF16>(maps, p, stream);
    case SOME_EPI_LN_GLU_BF16: return launch_gemm<SOME_EPI_LN_GLU_BF16>(maps, p, stream);
    case SOME_EPI_RESID_F32_LN: return launch_gemm<SOME_EPI_RESID_F32_LN>(maps, p, stream);
    case SOME_EPI_GLU_RESID_F32_LN: return launch_gemm<SOME_EPI_GLU_RESID_F32_LN>(maps, p, stream);
    case SOME_EPI_BIAS_F32: return launch_gemm<SOME_EPI_BIAS_F32>(maps, p, stream);
    case SOME_EPI_SIGMOID_F32: return launch_gemm<SOME_EPI_SIGMOID_F32>(maps, p, stream);
    case SOME_EPI_SOFTMAX_F32: return launch_gemm<SOME_EPI_SOFTMAX_F32>(maps, p, stream);
    default: SOME_REQUIRE(false, "some_gemm: unknown epilogue %d", epi);
  }
  return -1;
}
