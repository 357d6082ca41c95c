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
//                   epilogue (bias / SiLU / GLU / residual / LayerNorm fold / sigmoid / softmax).
// Epilogue stores: the bf16 and residual epilogues leave through shared memory.  Each consumer warpgroup fills slabs of
// 64 rows x 128 B (64 bf16 or 32 fp32 columns, 128-byte swizzle) and one thread sends each slab with a TMA store; the
// residual epilogues first TMA-load the residual slab (the next slab loads while this one is worked on) and add into it
// in place.  The head epilogues (ragged N) store straight from the accumulator registers.
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
constexpr int GEMM_THREADS = 384;
constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;   // 16 KB
constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;   // 32 KB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int ACC = BLOCK_N / 2;   // accumulator registers per consumer thread
constexpr int SLAB_ROWS = 64;      // epilogue slab: the rows of one consumer warpgroup ...
constexpr int SLAB_BYTES = SLAB_ROWS * 128;   // ... by 128 B (one 128-byte swizzle row)

struct GemmGroup {
  const float* bias;   // [N] in packed-column order, or nullptr
  void* out;           // head epilogues: f32, row pitch ld_out elements (the others store through GemmMaps::out)
  const float* ln_s;   // LayerNorm-folded consumers: column sums of W' [N]
  float* ln_stats;     // f32 [M][SOME_LN_SLOTS][2] partial (sum x, sum x^2): written by producers, read by consumers
};

// Tensor maps of one group.  resid / out: f32 boxes of 64 x 32 (residual epilogues) or bf16 boxes of 64 x 64 (out of
// the bf16 epilogues); out_bf16: bf16 64 x 64 (LayerNorm producers).  Maps an epilogue does not use are zero.
struct GemmMaps {
  CUtensorMap a, b, resid, out, out_bf16;
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
  static constexpr bool STAGED = BASE <= SOME_EPI_GLU_RESID_F32;   // everything but the heads goes through slabs
  static constexpr bool RESID = BASE == SOME_EPI_RESID_F32 || BASE == SOME_EPI_GLU_RESID_F32;
  static constexpr bool GLU = BASE == SOME_EPI_GLU_BF16 || BASE == SOME_EPI_GLU_RESID_F32;
  static constexpr int ELEM = RESID ? 4 : 2;            // bytes per output element in the slab
  static constexpr int SLAB_COLS = 128 / ELEM;
  static constexpr int SLABS = STAGED ? (GLU ? BLOCK_N / 2 : BLOCK_N) / SLAB_COLS : 0;   // per warpgroup and tile
  // Slab buffers per consumer warpgroup: two, so that one is filled (or loaded) while the other is stored.  The
  // LayerNorm producers add two bf16 slabs for the copy of out; they do not fit beside a 4-stage ring, and 64-byte
  // (32-column) bf16 slabs would need a second swizzle mode in the maps and the fragment mapping, so those two epilogues
  // run a 3-stage ring instead (ln_fold only; K = 512 gives 8 k-blocks per tile).
  static constexpr int SLAB_BUFS = !STAGED ? 0 : LNP ? 4 : 2;
  static constexpr int STAGES = LNP ? 3 : 4;
  static constexpr int SMEM = STAGES * STAGE_BYTES + 2 * SLAB_BUFS * SLAB_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(SMEM <= 232448, "gemm_kernel: shared memory over the 227 KB per-CTA limit");
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

// Slab state of one consumer warpgroup: its SLAB_BUFS buffers (0-1 staging, 2-3 the LayerNorm producers' bf16 copy),
// the mbarriers of the residual loads into buffers 0-1, the number of slabs it has used so far (buffer = count & 1,
// barrier parity = (count >> 1) & 1), and whether this thread is the one that issues the warpgroup's TMA operations
// (always the same thread: bulk groups belong to the thread that commits them).
struct Slabs {
  uint8_t* buf;
  uint64_t* bar;
  uint32_t count;
  bool leader;
};

// Shared address of this thread's columns 2 q, 2 q + 1 in slab row r, in the 128-byte swizzle of the tensor maps (the
// 16-byte chunk index is XORed with r % 8).  Column 8 u + 2 q of the row is then at slab_row(...) ^ (8 u * ELEM): the
// constant only flips chunk bits 4-6 (8 u * ELEM < 128), so one base per slab and row serves every column group, and
// the row r + 8 is at + 1024 (same r % 8).  The 8 rows of a warp (r % 8 = lane / 4) put one 8-column group into 8
// different chunks: a warp's bf16 stores hit 32 distinct banks, its fp32 pairs (256 B) each bank twice.
template <int ELEM>
__device__ __forceinline__ uint32_t slab_row(const uint8_t* slab, int r, int q) {
  constexpr int Q = 2 * ELEM;   // bytes per column pair
  return smem_u32(slab) + r * 128 + ((((Q * q) >> 4) ^ (r & 7)) << 4) + ((Q * q) & 15);
}

// Sends a residual slab's load (buffer count & 1).  Called by the leader only.
__device__ __forceinline__ void slab_load(const GemmMaps& tm, const Slabs& sl, uint32_t count, int col, int row) {
  uint64_t* bar = &sl.bar[count & 1];
  mbar_arrive_expect_tx(bar, SLAB_BYTES);   // rows past M are zero-filled and still counted
  tma_load_2d(sl.buf + (count & 1) * SLAB_BYTES, &tm.resid, bar, col, row);
}

// Staged epilogue of one consumer warpgroup (64 rows x 256 accumulator columns of the tile, starting at row_base):
// output columns are cut into Cfg::SLABS slabs of SLAB_COLS.  Per slab: (residual: wait for its TMA load, start the
// next one), each thread writes its values into the slab (in place: alpha * (acc + bias) + resid), fence.proxy.async,
// named barrier over the warpgroup, one TMA store.  Rows past M are clipped by the store.  The residual slab is read and
// written by this warpgroup only, and its load completes before its store is issued, so resid may alias out.
template <int EPI>
__device__ __forceinline__ void epilogue_staged(const GemmParams& p, const GemmGroup& g, const GemmMaps& tm,
                                                float (&acc)[ACC], Slabs& sl, int row_base, int lrow, int col_tile,
                                                int q, int cw) {
  using Cfg = EpiCfg<EPI>;
  constexpr int BASE = Cfg::BASE;
  constexpr int SC = Cfg::SLAB_COLS;
  const int col_out = Cfg::GLU ? col_tile / 2 : col_tile;   // first output column of the tile
  [[maybe_unused]] float st_s[2] = {}, st_q[2] = {};   // [row half]: (sum x, sum x^2) of the current ln_stats slot
#pragma unroll
  for (int c = 0; c < Cfg::SLABS; ++c) {
    const uint32_t count = sl.count + c;
    uint8_t* buf = sl.buf + (count & 1) * SLAB_BYTES;
    [[maybe_unused]] uint8_t* buf16 = sl.buf + (2 + ((count >> 1) & 1)) * SLAB_BYTES;   // LN producers: 2 slabs per copy
    if constexpr (Cfg::RESID) {
      mbar_wait(&sl.bar[count & 1], (count >> 1) & 1);
      if (sl.leader) {
        bulk_wait_group_read<0>();   // the previous slab's store has read the other buffer
        if (c + 1 < Cfg::SLABS) slab_load(tm, sl, count + 1, col_out + (c + 1) * SC, row_base);
      }
    }
    const uint32_t row = slab_row<Cfg::ELEM>(buf, lrow, q);
    [[maybe_unused]] const uint32_t row16 = slab_row<2>(buf16, lrow, q);
#pragma unroll
    for (int u = 0; u < SC / 8; ++u) {
      // 8-column output group og of the warpgroup -> accumulator group j (GLU: "out" half of packed group og / 2)
      const int og = c * (SC / 8) + u;
      const int j = Cfg::GLU ? 4 * (og >> 1) + (og & 1) : og;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t addr = (row ^ (8 * u * Cfg::ELEM)) + 1024 * h;
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if constexpr (BASE == SOME_EPI_SILU_BF16) v0 = silu_fast(v0), v1 = silu_fast(v1);
        if constexpr (Cfg::GLU) {
          v0 *= sigmoid_fast(acc[4 * (j + 2) + 2 * h]);
          v1 *= sigmoid_fast(acc[4 * (j + 2) + 2 * h + 1]);
        }
        if constexpr (Cfg::RESID) {
          const float2 rs = lds_f2(addr);
          float2 x;
          if constexpr (Cfg::GLU) x = make_float2(rs.x + v0, rs.y + v1);
          else x = make_float2(fmaf(v0, p.alpha, rs.x), fmaf(v1, p.alpha, rs.y));   // alpha * (acc + bias) + resid
          sts_f2(addr, x);
          if constexpr (Cfg::LNP) {
            st_s[h] += x.x + x.y;
            st_q[h] = fmaf(x.x, x.x, fmaf(x.y, x.y, st_q[h]));
            sts_u32((row16 ^ (2 * ((c & 1) * SC + 8 * u))) + 1024 * h, pack_bf16x2(x.x, x.y));
          }
        } else {
          sts_u32(addr, pack_bf16x2(v0, v1));
        }
      }
    }
    fence_proxy_async_smem();   // this thread's slab writes -> visible to the TMA store
    if constexpr (!Cfg::RESID)
      if (sl.leader) bulk_wait_group_read<0>();   // the previous slab's store has read the buffer the next slab fills
    named_bar_sync(1 + cw, 128);
    if (sl.leader) {
      tma_store_2d(&tm.out, buf, col_out + c * SC, row_base);
      if constexpr (Cfg::LNP)
        if (c & 1) tma_store_2d(&tm.out_bf16, buf16, col_out + (c - 1) * SC, row_base);
      bulk_commit_group();
    }
    if constexpr (Cfg::LNP) {
      // slot j / 16 of the tile (128 accumulator columns) is complete after its last slab
      constexpr int G8 = SC / 8;
      const int slot = (Cfg::GLU ? 4 * ((c * G8) >> 1) : c * G8) >> 4;
      const int next = (Cfg::GLU ? 4 * (((c + 1) * G8) >> 1) : (c + 1) * G8) >> 4;
      if (c + 1 == Cfg::SLABS || next != slot) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row_base + lrow + 8 * h;
          const float sum = quad_sum(st_s[h]), sq = quad_sum(st_q[h]);
          if (q == 0 && row < p.M)
            reinterpret_cast<float2*>(g.ln_stats)[(size_t)row * SOME_LN_SLOTS + (col_tile >> 7) + slot] = make_float2(sum, sq);
          st_s[h] = st_q[h] = 0.f;
        }
      }
    }
  }
  sl.count += Cfg::SLABS;
}

// Epilogue of one consumer thread: acc holds rows row0 and row0 + 8, columns col_tile + 8 j + 2 q + {0, 1} (j < 32),
// where row0 = row_base + lrow.
// GLU: packed columns come in 32-column groups [16 "out" | 16 "gate"], so the gate of acc[4 j + i] is acc[4 (j + 2) + i]
// (j % 4 < 2) and output channel (col_tile + 32 G) / 2 + 8 jj + 2 q + e belongs to group G, j = 4 G + jj.
// LayerNorm producers: slot col / 128 of ln_stats gets (sum x, sum x^2) of the row over those 128 accumulator columns.
template <int EPI>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, const GemmGroup& g, const GemmMaps& tm,
                                              float (&acc)[ACC], Slabs& sl, int row_base, int lrow, int col_tile, int q,
                                              int cw) {
  using Cfg = EpiCfg<EPI>;
  constexpr int BASE = Cfg::BASE;
  const int rows[2] = {row_base + lrow, row_base + lrow + 8};
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

  if constexpr (Cfg::STAGED) {
    epilogue_staged<EPI>(p, g, tm, acc, sl, row_base, lrow, col_tile, q, cw);
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
gemm_kernel(const __grid_constant__ GemmMaps tm0, const __grid_constant__ GemmMaps tm1, const GemmParams p) {
  using Cfg = EpiCfg<EPI>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* slabs = smem + STAGES * STAGE_BYTES;                                           // [2][SLAB_BUFS] slabs
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(slabs + 2 * Cfg::SLAB_BUFS * SLAB_BYTES);   // [STAGES]
  uint64_t* empty_bar = full_bar + STAGES;                                                // [STAGES]
  uint64_t* slab_bar = empty_bar + STAGES;                                                // [2][2] residual loads

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  const int num_m = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int num_n = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int tiles_per_group = num_m * num_n;
  const int num_tiles = tiles_per_group * p.groups;
  const int num_kb = (p.K + BLOCK_K - 1) / BLOCK_K;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.groups; ++i) {
      const GemmMaps* tm = i == 0 ? &tm0 : &tm1;
      tma_prefetch_desc(&tm->a);
      tma_prefetch_desc(&tm->b);
      if constexpr (Cfg::RESID) tma_prefetch_desc(&tm->resid);
      if constexpr (Cfg::STAGED) tma_prefetch_desc(&tm->out);
    }
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);   // one arrival per consumer warp
    }
    for (int i = 0; i < 4; ++i) mbar_init(&slab_bar[i], 1);
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
        const GemmMaps* tm = grp == 0 ? &tm0 : &tm1;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);   // out-of-bounds rows are zero-filled and still counted
          uint8_t* sa = smem + stage * STAGE_BYTES;
          tma_load_2d(sa, &tm->a, &full_bar[stage], kb * BLOCK_K, m_blk * BLOCK_M);
          tma_load_2d(sa + A_BYTES, &tm->b, &full_bar[stage], kb * BLOCK_K, n_blk * BLOCK_N);
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
    Slabs sl{slabs + cw * Cfg::SLAB_BUFS * SLAB_BYTES, slab_bar + 2 * cw, 0u, (threadIdx.x & 127) == 0};
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int grp = tile / tiles_per_group;
      const int t = tile - grp * tiles_per_group;
      const int m_blk = t / num_n, n_blk = t - m_blk * num_n;
      const GemmMaps* tm = grp == 0 ? &tm0 : &tm1;
      const int row_base = m_blk * BLOCK_M + cw * SLAB_ROWS;
      // the tile's first residual slab loads while the MMAs run (its buffer's last store was waited for, .read, in the
      // previous tile's last slab)
      if constexpr (Cfg::RESID)
        if (sl.leader) slab_load(*tm, sl, sl.count, Cfg::GLU ? n_blk * BLOCK_N / 2 : n_blk * BLOCK_N, row_base);
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
      epilogue_tile<EPI>(p, g, *tm, acc, sl, row_base, (warp & 3) * 16 + (lane >> 2), n_blk * BLOCK_N, lane & 3, cw);
    }
    // all stores performed before the CTA exits: a dependent kernel (programmatic launch) may read them at once
    if constexpr (Cfg::STAGED)
      if (sl.leader) bulk_wait_group<0>();
  }
}

template <int EPI>
static int launch_gemm(const GemmMaps* maps, const GemmParams& p, cudaStream_t stream) {
  auto kern = gemm_kernel<EPI>;
  constexpr int smem = EpiCfg<EPI>::SMEM;
  static bool configured[kMaxDevices] = {};   // function attributes are per device
  const int dev_ = device_index();
  if (!configured[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    SOME_REQUIRE(e == cudaSuccess, "cudaFuncSetAttribute(gemm, %d B smem): %s", smem, cudaGetErrorString(e));
    configured[dev_] = true;
  }
  const int num_m = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int num_n = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int tiles = num_m * num_n * p.groups;
  int grid = num_sms();
  if (tiles < grid) grid = tiles;
  launch_pdl(kern, dim3(grid), dim3(GEMM_THREADS), smem, stream, maps[0], maps[1], p);
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
  GemmMaps maps[2];
  memset(maps, 0, sizeof(maps));
  const auto aligned16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  for (int g = 0; g < 2; ++g) {
    const int s = g < a->groups ? g : 0;
    SOME_REQUIRE(a->A[s] != nullptr && a->W[s] != nullptr && a->out[s] != nullptr, "some_gemm: null pointer in group %d", s);
    if (make_tmap_bf16_2d(&maps[g].a, a->A[s], a->M, a->K, a->lda, BLOCK_M)) return -1;
    if (make_tmap_bf16_2d(&maps[g].b, a->W[s], a->N, a->K, a->K, BLOCK_N)) return -1;
    p.g[g].bias = a->bias[s];
    p.g[g].out = a->out[s];
    p.g[g].ln_s = a->ln_s[s];
    p.g[g].ln_stats = a->ln_stats[s];
    // the staged epilogues store (and the residual ones load) through tensor maps: 16-byte aligned bases and pitches
    if (needs_resid) {
      const int out_cols = glu_resid ? a->N / 2 : a->N;
      SOME_REQUIRE(a->resid[s] != nullptr, "some_gemm: epilogue %d needs a residual pointer (group %d)", epi, s);
      SOME_REQUIRE(a->ld_out % 4 == 0 && out_cols <= a->ld_out, "some_gemm: bad ld_out %d for %d output columns", a->ld_out, out_cols);
      SOME_REQUIRE(aligned16(a->resid[s]) && aligned16(a->out[s]),
                   "some_gemm: resid and out must be 16-byte aligned (group %d)", s);
      if (make_tmap_2d(&maps[g].resid, 4, a->resid[s], a->M, out_cols, a->ld_out, SLAB_ROWS, 32)) return -1;
      if (make_tmap_2d(&maps[g].out, 4, a->out[s], a->M, out_cols, a->ld_out, SLAB_ROWS, 32)) return -1;
      if (ln_producer) {
        SOME_REQUIRE(a->out_bf16[s] != nullptr && a->ln_stats[s] != nullptr,
                     "some_gemm: LayerNorm producer epilogue %d needs out_bf16 and ln_stats (group %d)", epi, s);
        SOME_REQUIRE(a->ld_out % 8 == 0 && aligned16(a->out_bf16[s]),
                     "some_gemm: out_bf16 needs a 16-byte aligned base and ld_out %% 8 == 0 (ld_out %d, group %d)",
                     a->ld_out, s);
        if (make_tmap_2d(&maps[g].out_bf16, 2, a->out_bf16[s], a->M, out_cols, a->ld_out, SLAB_ROWS, 64)) return -1;
      }
    }
    if (!head && !needs_resid) {
      const int out_cols = (epi == SOME_EPI_GLU_BF16 || epi == SOME_EPI_LN_GLU_BF16) ? a->N / 2 : a->N;
      SOME_REQUIRE(a->ld_out % 8 == 0 && out_cols <= a->ld_out, "some_gemm: bad ld_out %d for %d bf16 output columns", a->ld_out, out_cols);
      SOME_REQUIRE(aligned16(a->out[s]), "some_gemm: out must be 16-byte aligned (group %d)", s);
      if (make_tmap_2d(&maps[g].out, 2, a->out[s], a->M, out_cols, a->ld_out, SLAB_ROWS, 64)) return -1;
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
