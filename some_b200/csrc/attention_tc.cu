// K-attn (wgmma): per-clip (var-len) multi-head self-attention softmax(Q K^T / 8) V, no mask, 8 heads x 64
// (base_attention.py:34-45; conform_blocke never forwards a mask: Gconform.py:83-84,133).
//
// Input: the fused to_q|to_kv GEMM output qkv bf16 [M, 1536] = [q | k | v] (heads 64-wide, contiguous);
// output bf16 [M, 512] = 'b h t c -> b t (h c)'.  No head-major copies are made: Q/K/V tiles are TMA boxes cut
// straight out of qkv.
//
// CTA = 128 query rows of one (clip, head), 64-key tiles; 2 CTAs per SM (81 KB smem each).
// Roles (288 threads):
//   warps 0-7   two consumer warpgroups, 64 query rows each (wgmma M = 64).  Per key tile:
//               S = Q K_j^T (wgmma m64n64k16 x4, both operands K-major in shared memory) into 32 fp32 registers,
//               online softmax in base 2 on the registers (row = a quad of lanes), P -> bf16 pairs that are already in
//               the register layout of a wgmma A operand, O += P V_j (wgmma m64n64k16 x4, A from registers, B = V MN-major)
//   warp 8      TMA producer: Q once, then (K_j, V_j) 64-key tiles into a 4-stage ring (128-B swizzle)
// Rows of K/V beyond the clip end are masked (p = 0); rows beyond M are zero-filled by TMA.
#include "host_common.h"
#include "sm90_ptx.cuh"

#include "../../include/some_b200.h"

namespace some {

constexpr int TC_BM = 128;                 // queries per CTA
constexpr int TC_BN = 64;                  // keys per tile
constexpr int TC_QTILE = 128 * 64 * 2;     // 16 KB
constexpr int TC_KTILE = TC_BN * 64 * 2;   // 8 KB (K or V tile)
constexpr int TC_STAGES = 4;
constexpr int TC_THREADS = 288;
constexpr int TC_BAR_BYTES = 256;
constexpr int TC_SMEM = 1024 /*align slack*/ + TC_QTILE + TC_STAGES * 2 * TC_KTILE + TC_BAR_BYTES;

struct AttnTcParams {
  __nv_bfloat16* out[2];
  const int32_t* cu_frames;
  int tiles_per_clip;
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__global__ void __launch_bounds__(TC_THREADS, 2)
attention_tc_kernel(const __grid_constant__ CUtensorMap tmq0, const __grid_constant__ CUtensorMap tmkv0,
                    const __grid_constant__ CUtensorMap tmq1, const __grid_constant__ CUtensorMap tmkv1,
                    const AttnTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + TC_QTILE;                                  // stage s: K at +s * 2 * KTILE, V right after it
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + TC_STAGES * 2 * TC_KTILE);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;                      // [TC_STAGES]
  uint64_t* kv_empty = kv_full + TC_STAGES;          // [TC_STAGES]
  static_assert(8 * (1 + 2 * TC_STAGES) <= TC_BAR_BYTES, "barrier block too small");

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int clip = blockIdx.x / p.tiles_per_clip;
  const int qt = blockIdx.x - clip * p.tiles_per_clip;
  const int row_begin = p.cu_frames[clip];
  const int T = p.cu_frames[clip + 1] - row_begin;
  const int q0 = qt * TC_BM;
  if (q0 >= T) return;  // whole CTA, before any barrier use
  const int head = blockIdx.y;
  const int grp = blockIdx.z;
  const CUtensorMap* tmq = grp == 0 ? &tmq0 : &tmq1;
  const CUtensorMap* tmkv = grp == 0 ? &tmkv0 : &tmkv1;
  const int n_tiles = (T + TC_BN - 1) / TC_BN;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(tmq);
    tma_prefetch_desc(tmkv);
    mbar_init(q_full, 1);
    for (int i = 0; i < TC_STAGES; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 8);   // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  griddep_launch();     // programmatic dependent launch (host_common.h): qkv is read only after the producing GEMM has completed
  griddep_wait();

  if (warp == 8) {
    if (elect_one_sync()) {
      mbar_arrive_expect_tx(q_full, TC_QTILE);
      tma_load_2d(sQ, tmq, q_full, head * 64, row_begin + q0);
      int s = 0;
      uint32_t ph = 0;
      for (int j = 0; j < n_tiles; ++j) {
        mbar_wait(&kv_empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&kv_full[s], 2 * TC_KTILE);
        uint8_t* dst = sKV + s * 2 * TC_KTILE;
        tma_load_2d(dst, tmkv, &kv_full[s], SOME_DIM + head * 64, row_begin + j * TC_BN);
        tma_load_2d(dst + TC_KTILE, tmkv, &kv_full[s], 2 * SOME_DIM + head * 64, row_begin + j * TC_BN);
        if (++s == TC_STAGES) s = 0, ph ^= 1;
      }
    }
    __syncwarp();
    return;
  }

  // ---- consumers: warpgroup cw owns query rows [64 cw, 64 cw + 64) of the tile; this thread rows r and r + 8 (quad = row)
  const int cw = warp >> 2;
  const int q = lane & 3;
  const int r = cw * 64 + (warp & 3) * 16 + (lane >> 2);
  const float c = 0.125f * 1.4426950408889634f;  // dim_head^-0.5 * log2(e)
  const uint64_t qdesc = gmma_desc_kmajor_sw128(smem_u32(sQ + cw * 64 * 128));
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // per row half: running maximum (raw score), partial row sum

  mbar_wait(q_full, 0);
  for (int j = 0; j < n_tiles; ++j) {
    const int s = j % TC_STAGES;
    mbar_wait(&kv_full[s], (j / TC_STAGES) & 1);
    const uint32_t k_addr = smem_u32(sKV + s * 2 * TC_KTILE);
    const uint64_t kdesc = gmma_desc_kmajor_sw128(k_addr);
    float sc[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64k16_ss(sc, qdesc + 2 * k, kdesc + 2 * k, k != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence(sc);

    // ---- online softmax: sc[4 jj + 2 h + e] = score of row r + 8 h, key 8 jj + 2 q + e of the tile
    const int valid = min(TC_BN, T - j * TC_BN);  // keys of this tile inside the clip
    if (valid < TC_BN) {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (8 * jj + 2 * q + e >= valid) sc[4 * jj + e] = sc[4 * jj + 2 + e] = -INFINITY;
    }
    uint32_t pa[4][4];   // P as the A operand of PV: k-slice kk = keys [16 kk, 16 kk + 16)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) mx = fmaxf(mx, fmaxf(sc[4 * jj + 2 * h], sc[4 * jj + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx);   // finite: every tile has at least one valid key
      const float alpha = ex2_approx((m_run[h] - m_new) * c);   // 0 on the first tile (-inf)
      m_run[h] = m_new;
      const float mc = m_new * c;
      float ts = 0.f;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const float p0 = ex2_approx(fmaf(sc[4 * jj + 2 * h], c, -mc));
        const float p1 = ex2_approx(fmaf(sc[4 * jj + 2 * h + 1], c, -mc));
        ts += p0 + p1;
        // A fragment of wgmma k16: regs {row r k 2q.., row r+8 k 2q.., row r k 8+2q.., row r+8 k 8+2q..}
        pa[jj >> 1][(jj & 1) * 2 + h] = pack_bf16x2(p0, p1);
      }
      l[h] = fmaf(l[h], alpha, ts);
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        o[4 * jj + 2 * h] *= alpha;
        o[4 * jj + 2 * h + 1] *= alpha;
      }
    }

    // ---- O += P V_j: 16 keys per MMA, B = V rows (keys) 16 kk .. : +2 KB
    const uint32_t v_addr = k_addr + TC_KTILE;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_m64n64k16_rs_tb(o, pa[kk], gmma_desc_mnmajor_sw128(v_addr + kk * 2048, 1024));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[s]);
  }

  // ---- O / l -> bf16 -> out[row, head * 64 ..]
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float lt = l[h];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    const float inv = 1.0f / lt;
    const int qrow = q0 + r + 8 * h;
    if (qrow < T) {
      __nv_bfloat16* dst = p.out[grp] + (size_t)(row_begin + qrow) * SOME_DIM + head * 64 + 2 * q;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
    }
  }
}

}  // namespace some

using namespace some;

extern "C" int some_attention_varlen(const some_attn_args* a, cudaStream_t stream) {
  SOME_REQUIRE(a != nullptr && (a->groups == 1 || a->groups == 2), "some_attention_varlen: bad args");
  if (a->B <= 0 || a->max_frames <= 0 || a->M <= 0) return 0;
  SOME_REQUIRE(a->cu_frames != nullptr, "some_attention_varlen: null cu_frames");
  AttnTcParams p;
  CUtensorMap maps[4];
  for (int g = 0; g < 2; ++g) {
    const int s = g < a->groups ? g : 0;
    SOME_REQUIRE(a->qkv[s] && a->out[s], "some_attention_varlen: null pointer in group %d", s);
    if (make_tmap_bf16_2d(&maps[2 * g], a->qkv[s], a->M, 3 * SOME_DIM, 3 * SOME_DIM, TC_BM)) return -1;
    if (make_tmap_bf16_2d(&maps[2 * g + 1], a->qkv[s], a->M, 3 * SOME_DIM, 3 * SOME_DIM, TC_BN)) return -1;
    p.out[g] = reinterpret_cast<__nv_bfloat16*>(a->out[s]);
  }
  p.cu_frames = a->cu_frames;
  p.tiles_per_clip = (a->max_frames + TC_BM - 1) / TC_BM;
  static bool configured[kMaxDevices] = {};   // function attributes are per device
  const int dev_ = device_index();
  if (!configured[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM);
    SOME_REQUIRE(e == cudaSuccess, "cudaFuncSetAttribute(attention_tc): %s", cudaGetErrorString(e));
    // two CTAs per SM need more than the default shared-memory carveout
    e = cudaFuncSetAttribute(attention_tc_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                             cudaSharedmemCarveoutMaxShared);
    SOME_REQUIRE(e == cudaSuccess, "cudaFuncSetAttribute(attention_tc carveout): %s", cudaGetErrorString(e));
    configured[dev_] = true;
  }
  const long long gx = 1ll * p.tiles_per_clip * a->B;
  SOME_REQUIRE(gx < (1ll << 31), "some_attention_varlen: grid too large");
  dim3 grid(static_cast<unsigned>(gx), SOME_HEADS, a->groups);
  launch_pdl(attention_tc_kernel, grid, dim3(TC_THREADS), TC_SMEM, stream, maps[0], maps[1], maps[2], maps[3], p);
  return check_launch("some_attention_varlen");
}
