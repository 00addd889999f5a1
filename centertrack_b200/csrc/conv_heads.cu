// Fused output heads on the halo engine: every head's 3x3 conv 64 -> mid_c (+ bias, ReLU, bf16) and its 1x1 conv
// mid_c -> C_out (+ bias, head activation, fp32 NCHW) in one persistent launch, so the mid_c-channel intermediate of
// all heads (1 GB per step at B = 32, 512 x 512, four heads) is never written to or read back from HBM.
//
//   * Work item = one 8 (x) x 16 (y) output tile = 128 GEMM rows; its 10 x 18 x 64-channel input halo arrives once by
//     TMA (128-byte swizzled pixel rows) and every 3x3 tap is a descriptor-shifted view of it, as in conv_halo.cu.
//   * Per tile, per head, per mid "half" of NH = 128 (mid_c 256) or 64 (mid_c 64) channels: the 3x3 chain (9 taps x
//     4 K=16 steps, M64 x NH per warpgroup) into registers, + bias, ReLU, bf16 -> the warpgroup's 64 x NH mid tile in
//     shared memory (128-byte swizzled K-major, the MMA's own A layout), then that half's K part of the head's 1x1
//     chain into a second accumulator that lives across the halves; after the last half the head's epilogue.
//     K order and instruction shapes are those of the unfused layers (heads.0 at N = NH, each head's 1x1 at its
//     n_tile), so the head maps are bit-identical to the two-pass plan.
//   * The weights of all heads (1.2 MB for four 256-channel heads) do not fit: they stream through a ring of 16 KB
//     slots in consumption order -- per (head, half) nine 3x3 slices of 4 K blocks x NH, then the half's 1x1 slices
//     of 4 K blocks x n_tile.
//
// Warp roles (320 threads): warps 0-7 are two warpgroups, each owning 64 rows of every tile; warp 8 streams the
// weight ring; warp 9 loads the halo tiles (two stages).
#include "conv_common.cuh"
#include "wgmma.cuh"
#include <cuda.h>

namespace ctb {

constexpr int HD_TW = 8, HD_TH = 16;      // output tile (x, y)
constexpr int HD_THREADS = 320;
constexpr int HD_HALO_STAGES = 2;
constexpr int HD_MAX_N2 = 80;             // widest 1x1 n_tile (the 80-class COCO heat map)
constexpr uint32_t HD_SLOT_BYTES = 16384; // one weight slice: 4 K blocks x 128 columns x 32 bytes
constexpr int HD_STAGING_BYTES = 2 * 64 * EPI_PITCH * 4;

struct HeadArgs {
  ConvGeom g;
  const unsigned char* w1;     // 3x3 weights, halo packing at n_tile = NH: [n_heads * halves][36 K blocks][NH x 32 B]
  const float* shift;          // [n_heads * mid_c] 3x3 bias
  int n_heads, halves, w_stages;
  int tiles_x, tiles_y, tiles_total;
  uint32_t halo_bytes, box_bytes;
  uint32_t a_ahi;              // A descriptor bits 32-63: SBO = one halo row, 128-byte swizzle
  uint32_t a_sky;              // descriptor start-address units (16 B) per halo row
  struct Head { const unsigned char* w2; const float* bias; float* out; int c_out, act; } h[CT_MAX_FUSED_HEADS];
};

// NH: mid channels per pass; N2: the 1x1 n_tile, one for all heads of the launch (a runtime choice between MMA
// shapes next to the asynchronous MMAs would make ptxas serialise them)
template <int NH, int N2>
__global__ void __launch_bounds__(HD_THREADS, 1)
conv_heads_kernel(const __grid_constant__ HeadArgs a, const __grid_constant__ CUtensorMap tmap) {
  extern __shared__ __align__(1024) unsigned char hsm_dyn[];
  unsigned char* sm = hsm_dyn + ((1024u - (smem_u32(hsm_dyn) & 1023u)) & 1023u);
  const ConvGeom& g = a.g;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int S = a.w_stages;
  constexpr uint32_t MID_BYTES = 64u * NH * 2u;     // one warpgroup's 64 rows x NH channels, 8 KB per 64 channels
  constexpr int KSL = NH / 64;                      // 1x1 weight slices per half

  // smem: [halo stages][weight ring][mid tile x 2 warpgroups][epilogue staging][barriers]
  const uint32_t base = smem_u32(sm);
  const uint32_t sH = base;
  const uint32_t sW = sH + HD_HALO_STAGES * a.halo_bytes;
  const uint32_t sM = sW + (uint32_t)S * HD_SLOT_BYTES;
  const uint32_t sS = sM + 2u * MID_BYTES;
  const uint32_t bars = sS + HD_STAGING_BYTES;
  auto halo_full = [&](int s) { return bars + 8u * s; };
  auto halo_empty = [&](int s) { return bars + 8u * (HD_HALO_STAGES + s); };
  auto w_full = [&](int s) { return bars + 8u * (2 * HD_HALO_STAGES + s); };
  auto w_empty = [&](int s) { return bars + 8u * (2 * HD_HALO_STAGES + S + s); };

  pdl_trigger();
  if (tid == 0) {
    for (int s = 0; s < HD_HALO_STAGES; ++s) { mbar_init(halo_full(s), 1); mbar_init(halo_empty(s), 8); }
    for (int s = 0; s < S; ++s) { mbar_init(w_full(s), 1); mbar_init(w_empty(s), 8); }
    mbar_init_fence();
  }
  __syncthreads();
  pdl_wait();
  const int per_img = a.tiles_x * a.tiles_y;

  if (warp == 8) {
    if (lane == 0) {
      // ===================== weight ring producer: slices in the order the warpgroups consume them =====================
      uint32_t k = 0;
      auto put = [&](const unsigned char* src, uint32_t bytes) {
        const int s = (int)(k % (uint32_t)S);
        mbar_wait(w_empty(s), ((k / (uint32_t)S) & 1u) ^ 1u, 4, (int)k);
        mbar_arrive_expect_tx(w_full(s), bytes);
        bulk_g2s(sW + (uint32_t)s * HD_SLOT_BYTES, src, bytes, w_full(s));
        ++k;
      };
      for (int sp = blockIdx.x; sp < a.tiles_total; sp += gridDim.x)
        for (int h = 0; h < a.n_heads; ++h) {
          for (int j = 0; j < a.halves; ++j) {
            const unsigned char* w1 = a.w1 + (size_t)(h * a.halves + j) * 36 * NH * 32;
            for (int t = 0; t < 9; ++t) put(w1 + t * 4 * NH * 32, 4u * NH * 32u);
            for (int q = 0; q < KSL; ++q) put(a.h[h].w2 + (size_t)(j * KSL + q) * 4 * N2 * 32, 4u * N2 * 32u);
          }
        }
    }
  } else if (warp == 9) {
    if (lane == 0) {
      // ===================== halo producer =====================
      int it = 0;
      for (int sp = blockIdx.x; sp < a.tiles_total; sp += gridDim.x, ++it) {
        const int s = it % HD_HALO_STAGES;
        mbar_wait(halo_empty(s), ((uint32_t)(it / HD_HALO_STAGES) & 1u) ^ 1u, 5, it);
        const int b = sp / per_img, r = sp - b * per_img;
        const int ty = r / a.tiles_x, tx = r - ty * a.tiles_x;
        mbar_arrive_expect_tx(halo_full(s), a.box_bytes);
        tma_4d(sH + (uint32_t)s * a.halo_bytes, &tmap, 0, tx * HD_TW - 1, ty * HD_TH - 1, b, halo_full(s));
      }
    }
  } else {
    // ===================== MMA + epilogue warpgroups =====================
    const int wg = warp >> 2, w4 = warp & 3;
    const int lrow = 32 * (w4 & 1) + lane;           // epilogue: row per thread
    const int chalf = w4 >> 1;                       // 16-column half of each 32-column chunk
    const int row = 64 * wg + lrow;                  // GEMM row = pixel (ty * 16 + row / 8, tx * 8 + row % 8)
    const int gy = row >> 3, rx = row & 7;
    const uint32_t stg = sS + (uint32_t)wg * (64u * EPI_PITCH * 4u);
    const uint32_t mid = sM + (uint32_t)wg * MID_BYTES;
    // accumulator fragment of this thread (wgmma.cuh): rows frow, frow + 8, columns 8 i + fcol, + 1
    const int fl = tid & 31, frow = 16 * w4 + (fl >> 2), fcol = 2 * (fl & 3);
    const uint32_t half16 = (uint32_t)wg * 8u * (a.a_ahi & 0x3FFFu);
    const uint64_t a_hi = (uint64_t)a.a_ahi << 32;
    // mid tile as the 1x1's A operand: 128-byte swizzle, K-major, SBO = 8 rows x 128 B
    const uint64_t mid_desc = wg_desc(mid, 16u, 1024u, 1u);
    const int HWo = g.OH * g.OW;
    // one arrival per warp, predicated rather than branched: MMAs are in flight
    auto release = [&](uint32_t kk, bool pred) {
      __syncwarp();
      mbar_arrive_if(w_empty((int)(kk % (uint32_t)S)), pred && lane == 0);
    };
    float acc[NH / 2];
    float acc2[N2 / 2];
    uint32_t k = 0;
    int it = 0;
    for (int sp = blockIdx.x; sp < a.tiles_total; sp += gridDim.x, ++it) {
      const int hs = it % HD_HALO_STAGES;
      mbar_wait(halo_full(hs), (uint32_t)(it / HD_HALO_STAGES) & 1u, 6, it);
      const uint32_t a_lo0 = (1u << 16) + ((sH + (uint32_t)hs * a.halo_bytes) >> 4) + half16;
      const int b = sp / per_img, r = sp - b * per_img;
      const int ty = r / a.tiles_x, tx = r - ty * a.tiles_x;
      const int oy = ty * HD_TH + gy, ox = tx * HD_TW + rx;
      const bool p_ok = oy < g.OH && ox < g.OW;
      for (int h = 0; h < a.n_heads; ++h) {
        for (int j = 0; j < a.halves; ++j) {
          // ---- 3x3 chain of this half: one weight slice per tap, the previous slice released once its MMAs are done.
          // A wgmma fence opens every slice's MMAs: without it ptxas inserts one after the wait and serialises them.
          for (int tap = 0; tap < 9; ++tap, ++k) {
            const int s = (int)(k % (uint32_t)S);
            mbar_wait_inline(w_full(s), (k / (uint32_t)S) & 1u);
            const uint32_t a_lo = a_lo0 + (uint32_t)(tap / 3) * a.a_sky + (uint32_t)(tap % 3) * 8u;
            const uint64_t b_desc = wg_desc(sW + (uint32_t)s * HD_SLOT_BYTES, NH * 16u, 128u, 0u);
            wg_fence();
#pragma unroll
            for (int q = 0; q < 4; ++q)
              Wgmma<NH>::mma(acc, a_hi | (uint64_t)(a_lo + 2u * q), b_desc + (uint64_t)q * ((NH * 32) >> 4),
                             (tap | q) != 0 ? 1u : 0u);
            wg_commit();
            wg_wait<1>();
            release(k - 1, tap > 0);
          }
          wg_wait<0>();
          wg_fence_operand(acc);
          release(k - 1, true);
          // the tile's last 3x3 chain: the halo stage is free
          mbar_arrive_if(halo_empty(hs), lane == 0 && h == a.n_heads - 1 && j == a.halves - 1);
          // ---- bf16(relu(acc + bias)) -> this warpgroup's mid tile.  Each warp writes the rows its own MMAs read,
          // and the previous half's 1x1 MMAs are complete (wait<0> below), so the tile is free.
          const float* sh = a.shift + (size_t)(h * a.halves + j) * NH;
#pragma unroll
          for (int i = 0; i < NH / 8; ++i) {
            const int c = 8 * i + fcol;
            const float s0 = __ldg(sh + c), s1 = __ldg(sh + c + 1);
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const int rr = frow + 8 * hh;
              const __nv_bfloat162 v = __floats2bfloat162_rn(fmaxf(acc[4 * i + 2 * hh] + s0, 0.f),
                                                            fmaxf(acc[4 * i + 2 * hh + 1] + s1, 0.f));
              const uint32_t addr = mid + (uint32_t)(i >> 3) * 8192u + (uint32_t)rr * 128u +
                                    ((uint32_t)((i & 7) ^ (rr & 7)) << 4) + (uint32_t)fcol * 2u;
              sts32(addr, *reinterpret_cast<const uint32_t*>(&v));
            }
          }
          fence_proxy_async();
          named_sync(1 + wg, 128);
          // ---- this half's K part of the head's 1x1 chain
          for (int q = 0; q < KSL; ++q, ++k) {
            const int s = (int)(k % (uint32_t)S);
            mbar_wait_inline(w_full(s), (k / (uint32_t)S) & 1u);
            const uint64_t ad = mid_desc + (uint64_t)(q * (8192 >> 4));
            const uint64_t bd = wg_desc(sW + (uint32_t)s * HD_SLOT_BYTES, N2 * 16u, 128u, 0u);
            wg_fence();
#pragma unroll
            for (int kq = 0; kq < 4; ++kq)
              Wgmma<N2>::mma(acc2, ad + 2u * kq, bd + (uint64_t)kq * ((N2 * 32) >> 4), (j | q | kq) != 0 ? 1u : 0u);
            wg_commit();
          }
          wg_wait<0>();
          wg_fence_operand(acc2);
          for (int q = 0; q < KSL; ++q) release(k - KSL + q, true);
        }
        // ---- head epilogue: + bias, activation, fp32 NCHW (the unfused 1x1 launch's epilogue)
        ConvGeom gh = g;
        gh.C_out = a.h[h].c_out; gh.relu = 0; gh.head_act = a.h[h].act;
        const float* bias = a.h[h].bias;
#pragma unroll
        for (int c0 = 0; c0 < N2; c0 += 32) {
          named_sync(1 + wg, 128);                    // the previous chunk's readers are done with the staging tile
          stage_acc_chunk(acc2, c0, stg, 0);
          named_sync(1 + wg, 128);
          const int col = c0 + chalf * 16;
          if (col >= N2 || !p_ok || col >= gh.C_out) continue;
          float v[16];
          lds_f(stg + (uint32_t)lrow * EPI_PITCH * 4u + (uint32_t)chalf * 64u, v);
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) v[jj] += col + jj < gh.C_out ? __ldg(bias + col + jj) : 0.f;
          store_head16(a.h[h].out + ((size_t)b * gh.C_out + col) * HWo + (size_t)oy * g.OW + ox, HWo, v, col, gh);
        }
      }
    }
  }
}

// ---- host ----
// Configuration step: the launch arguments other than the pointers, and the launch configuration.  No CUDA call.
static int heads_config(const ct_conv_desc* d, HeadArgs& a, ConvConfig& c) {
  a.g = make_geom(d);
  const ConvGeom& g = a.g;
  if (g.KH != 3 || g.KW != 3 || g.stride != 1 || g.pad != 1 || g.OH != g.H || g.OW != g.W)
    return fail(CT_ERR_INVALID, "fused heads: the shared layer must be a 3x3 stride-1 'same' convolution%s", "");
  if (g.C_in != 64 || g.ld_in % 8 != 0)
    return fail(CT_ERR_INVALID, "fused heads: C_in must be 64 (ld_in %% 8 == 0)%s (%ld)", "", g.C_in);
  if (d->n_heads < 1 || d->n_heads > CT_MAX_FUSED_HEADS || !d->heads)
    return fail(CT_ERR_INVALID, "fused heads: 1 .. 12 heads and a head table%s (%ld)", "", d->n_heads);
  if (g.C_out % d->n_heads != 0 || !(g.C_out / d->n_heads == 64 || g.C_out / d->n_heads == 256))
    return fail(CT_ERR_INVALID, "fused heads: 64 or 256 mid channels per head%s (C_out %ld)", "", g.C_out);
  const int mid_c = g.C_out / d->n_heads;
  if (d->n_tile != (mid_c == 256 ? 128 : 64))
    return fail(CT_ERR_INVALID, "fused heads: n_tile must be 128 (256 mid channels) or 64 (64)%s (%ld)", "", d->n_tile);
  if (g.out_mode != CT_OUT_NCHW_F32 || !g.relu || d->residual || d->epilogue_sum3)
    return fail(CT_ERR_INVALID, "fused heads: fp32 NCHW outputs, ReLU on the 3x3, no residual%s", "");
  a.n_heads = d->n_heads;
  a.halves = mid_c / d->n_tile;
  for (int i = 0; i < d->n_heads; ++i) {
    const ct_head& hd = d->heads[i];
    if (hd.C_out < 1 || hd.n_tile % 16 != 0 || hd.n_tile < hd.C_out || hd.n_tile > HD_MAX_N2 ||
        hd.n_tile != d->heads[0].n_tile)
      return fail(CT_ERR_INVALID, "fused heads: one n_tile for every head, C_out <= n_tile <= 80, n_tile %% 16 == 0%s (head %ld)", "", i);
    a.h[i].c_out = hd.C_out; a.h[i].act = hd.head_act;
    a.h[i].w2 = (const unsigned char*)hd.w; a.h[i].bias = hd.bias; a.h[i].out = hd.out;
  }
  const int pw = HD_TW + 2, ph = HD_TH + 2;
  a.box_bytes = (uint32_t)(pw * ph * 128);
  a.halo_bytes = (a.box_bytes + 1023u) & ~1023u;
  a.a_sky = (uint32_t)pw * 8u;
  a.a_ahi = a.a_sky | (1u << 30);
  a.tiles_x = (g.OW + HD_TW - 1) / HD_TW;
  a.tiles_y = (g.OH + HD_TH - 1) / HD_TH;
  a.tiles_total = g.B * a.tiles_x * a.tiles_y;
  auto smem_for = [&](int s) {
    return (size_t)HD_HALO_STAGES * a.halo_bytes + (size_t)s * HD_SLOT_BYTES + 2u * 64u * d->n_tile * 2u +
           HD_STAGING_BYTES + 1024 + 1024;
  };
  // the deepest weight ring that fits: both warpgroups read every slice, so the lead one may run that far ahead
  int stages = 0;
  for (int s = 8; s >= 3 && !stages; --s)
    if (smem_for(s) <= 227 * 1024) stages = s;
  if (!stages) return fail(CT_ERR_UNSUPPORTED, "fused heads: shared memory%s", "");
  a.w_stages = stages;
  c.smem_bytes = (int32_t)smem_for(stages);
  c.stages = stages;
  c.tile_w = HD_TW;
  c.tile_h = HD_TH;
  c.ctas_per_sm = 1;
  c.overlap = 0;
  return CT_OK;
}

int conv_config_heads(const ct_conv_desc* d, ConvConfig* c) {
  HeadArgs a;
  return heads_config(d, a, *c);
}

int conv_forward_heads(const ct_conv_desc* d, cudaStream_t st) {
  HeadArgs a;
  ConvConfig c;
  const int rc = heads_config(d, a, c);
  if (rc != CT_OK) return rc;
  if (((uintptr_t)d->x & 15) || ((uintptr_t)d->w & 15) || !d->shift)
    return fail(CT_ERR_INVALID, "fused heads: x / w must be 16-byte aligned, shift given%s", "");
  for (int i = 0; i < d->n_heads; ++i)
    if (!d->heads[i].w || ((uintptr_t)d->heads[i].w & 15) || !d->heads[i].bias || !d->heads[i].out)
      return fail(CT_ERR_INVALID, "fused heads: every head needs 16-byte aligned w, bias and out%s (head %ld)", "", i);
  a.w1 = (const unsigned char*)d->w;
  a.shift = d->shift;
  const ConvGeom& g = a.g;
  CUtensorMap tmap;
  const cuuint64_t dims[4] = {(cuuint64_t)g.C_in, (cuuint64_t)g.W, (cuuint64_t)g.H, (cuuint64_t)g.B};
  const cuuint64_t strides[3] = {(cuuint64_t)g.ld_in * 2, (cuuint64_t)g.W * g.ld_in * 2,
                                 (cuuint64_t)g.H * g.W * g.ld_in * 2};
  const cuuint32_t box[4] = {64, (cuuint32_t)(HD_TW + 2), (cuuint32_t)(HD_TH + 2), 1};
  const int r = encode_tmap_bf16(&tmap, d->x, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
  if (r != CT_OK) return r;
  const int grid = device_sm_count() < a.tiles_total ? device_sm_count() : a.tiles_total;
  return dispatch_n_tile(d->heads[0].n_tile, [&](auto n) {
    constexpr int N2 = decltype(n)::value;
    if constexpr (N2 <= HD_MAX_N2) {
      if (d->n_tile == 128)
        return launch_big_smem<conv_heads_kernel<128, N2>>(dim3(grid), dim3(HD_THREADS), c.smem_bytes, st, a, tmap);
      return launch_big_smem<conv_heads_kernel<64, N2>>(dim3(grid), dim3(HD_THREADS), c.smem_bytes, st, a, tmap);
    }
    return fail(CT_ERR_INVALID, "fused heads: n_tile%s", "");
  });
}

}  // namespace ctb
