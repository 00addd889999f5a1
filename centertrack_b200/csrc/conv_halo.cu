// "Halo" wgmma convolution for stride-1 KxK layers whose weights fit in shared memory (C_in 8..256):
// the im2row-free design for the thin, high-resolution layers (stems, level0, the 64-channel 128x128
// layers, DCN offset convs, the fused head 3x3) where a per-tap gather is LSU-bound.
//
//   * Output tile = 8 (x) x 16 (y) pixels = 128 GEMM rows (32 x 4 for 1x1 convs writing NCHW planes).  Its input
//     neighbourhood (tile + halo) is fetched ONCE by TMA tensor copies (cp.async.bulk.tensor.4d, zero fill
//     outside the image = the conv's zero padding).  Staging modes: whole-pixel K-major rows of 32/64/128 bytes
//     with the matching hardware swizzle (C_in 16/32/64, and 64-channel chunks for C_in 128..256) -- one TMA
//     request per pixel row; C_in == 8 (the packed stem input): 16-byte rows, two taps paired in one K=16 MMA;
//     un-swizzled 8-channel "planes" [halo_y][halo_x][8] (C_in 48, and debug: CTB_HALO_MODE=planes).
//   * NO data is rearranged per tap: the A operand of tap (ky,kx) is the same shared-memory tile addressed
//     through a wgmma descriptor whose start address is shifted by (ky*pitch + kx) pixel rows (the MMA's swizzle is
//     a function of the shared-memory address, like the TMA's, so a shifted start needs no base-offset field);
//     SBO = halo row pitch: the next 8-row core-matrix group is the next tile row.
//   * Weights of one output-channel tile stay resident in shared memory for the CTA's lifetime
//     (persistent CTAs, static tile striding); 2-4 halo stages so the TMA of the next tiles overlaps this one.
//
// Warp roles (288 threads): warps 0-7 are two warpgroups; warpgroup w issues the wgmma chain (M=64, N=n_tile, K=16
// per block) of GEMM rows 64w..64w+63 of every tile and then runs that half's epilogue (accumulator -> shared memory,
// 32 columns at a time -> row-per-thread stores).  Warp 8 is the TMA producer.  Two CTAs per SM where shared memory
// allows, so one CTA's epilogue overlaps the other's MMAs; where only one fits and 64 <= N <= 128, the two warpgroups
// take turns on the tensor cores instead (ping-pong), so one warpgroup's epilogue overlaps the other's MMAs.
//
// Pixel-major flavour (n_tile == C_out == 64, NHWC bf16 output): an m64n64k16 reads 2 KB of A and 2 KB of B from shared
// memory per 32 tensor-core cycles, the whole shared-memory bandwidth.  There the operands swap: A = the weights of the
// K16 block (64 output channels, the same packed blocks through the same descriptor B uses otherwise), B = the item's
// 128 halo pixel rows (the pixel-row descriptor above, whole tile: N = 128 is 16 core-matrix groups at SBO = pitch),
// one m64n128k16 per block, 96 B/cycle.  A warpgroup then takes whole items (warpgroup w: items w, w + 2, ...), its
// accumulator is [64 channels][128 pixels], and its epilogue transposes it through the staging tile 32 pixels at a
// time.  The walk (ky, kx, chunk, K-step) is a compile-time PxWalk, so the chain unrolls.
#include "conv_common.cuh"
#include "wgmma.cuh"
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

namespace ctb {

constexpr int HT_W = 8, HT_H = 16;       // output tile (x, y)

// Optional timeline trace of CTA 0 (ct_debug_trace): 8 clock64() stamps per work item --
// 0 producer acquired the halo stage, 1 TMA issued, 2 MMA saw the halo, 4 MMAs complete, 5 epilogue started,
// 6 epilogue done.  Off (nullptr) by default.
__device__ unsigned long long* g_halo_trace = nullptr;
// The pointer is read once per thread at kernel entry: a stamp must not cost a dependent load when tracing is off.
__device__ __forceinline__ unsigned long long* h_trace_ptr() {
  unsigned long long* t = g_halo_trace;
  return (t != nullptr && blockIdx.x == 0) ? t : nullptr;
}
__device__ __forceinline__ void h_stamp(unsigned long long* t, int it, int k) {
  if (t != nullptr && it < 256) t[it * 8 + k] = (unsigned long long)clock64();
}
constexpr int H_THREADS = 288;           // 2 MMA / epilogue warpgroups + TMA warp
constexpr int H_MMA_WARPS = 8;
constexpr int H_STAGING_BYTES = 2 * 64 * EPI_PITCH * 4;

struct HaloArgs {
  ConvGeom g;
  const __nv_bfloat16* w;       // packed blocks (see ct_pack_weights, engine HALO)
  const float* shift;
  const __nv_bfloat16* residual;
  void* out;
  int n_tile, n_tiles_n, nblk, planes, pw, ph, plane_bytes, box_bytes, halo_stages;
  int tw, th;                           // output tile: 8 x 16, or 32 x 4 for 1x1 convs writing NCHW planes
  int tiles_x, tiles_y, tiles_total;    // spatial tiles per image / total work items (incl. n tiles)
  int pair_taps;                        // 1: C_in == 8, one MMA = taps (kx, kx+1)
  int swz;                              // 0: un-swizzled 8-channel planes; else row bytes (32/64/128): whole
                                        //    pixel (all C_in channels) per K-major row, hardware swizzle
  int merged_xc;                        // 1: 3-D tensor map with (x, c) merged (C_in == ld_in == 8)
  int out_s2d;                          // CT_OUT_NHWC_S2D: pixel index remapped in the epilogue (g.out_mode = CT_OUT_NHWC)
  int sum3;                             // != 0: stem epilogue sum_g relu(group g + shift) -> 16 ch; bit g = group present
  uint32_t w_bytes;                     // bytes of one n-tile's weights
  // A-descriptor walk of one work item (all in 16-byte units, warp-uniform): for ky, kx|pair, chunk, kstep
  int m_nky, m_nkx, m_nc, m_nq;
  uint32_t m_sky, m_skx, m_sc, m_sq, m_alo, m_ahi;
  int px;                               // != 0: pixel-major flavour, the PX_WALKS entry (1-based) of its walk
};

// Compile-time walk of the pixel-major chain: KY x KX taps, NC 64-channel chunks, NQ K16 steps per chunk
template <int KY, int KX, int NC, int NQ>
struct PxWalk {
  static constexpr bool on = true;
  static constexpr int ky = KY, kx = KX, nc = NC, nq = NQ;
};
struct NoPx {
  static constexpr bool on = false;
  static constexpr int ky = 0, kx = 0, nc = 0, nq = 0;
};
// (KH, KW, C_in) of the 64 -> 64-channel layers of the shipped plans: level0 and the level2 3x3s (3x3, 64),
// level2.tree1.conv1 on level1's space-to-depth output (2x2, 128), level2.project (1x1, 32) and level2's root (1x1, 128)
constexpr int PX_WALKS[][3] = {{3, 3, 64}, {2, 2, 128}, {1, 1, 32}, {1, 1, 128}};
constexpr int PX_PITCH = 68;      // floats per pixel row of the pixel-major staging tile (32 x 64 channels + pad)

// OVERLAP: the flavour for launches that get one CTA per SM (64 <= N <= 128): the warpgroups' MMA chains alternate (see
// the item loop) and the register cap is that of one CTA.
// PX: the pixel-major flavour's walk (N == 64), or NoPx.
template <int N, bool OVERLAP, class PX = NoPx>
__global__ void __launch_bounds__(H_THREADS, (N <= 128 && !OVERLAP) ? 2 : 1)
conv_halo_kernel(const HaloArgs a, const __grid_constant__ CUtensorMap tmap) {
  extern __shared__ __align__(1024) unsigned char hsm_dyn[];
  unsigned char* sm = hsm_dyn + ((1024u - (smem_u32(hsm_dyn) & 1023u)) & 1023u);
  const ConvGeom& g = a.g;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  unsigned long long* const trace = h_trace_ptr();
  const int S = a.halo_stages;
  const uint32_t halo_bytes = (uint32_t)a.planes * a.plane_bytes;

  // smem: [weights][halo stage 0..S-1][epilogue staging 2 x 64 x 36 fp32][barriers][shift]
  const uint32_t base = smem_u32(sm);
  const uint32_t sW = base;
  const uint32_t sH = base + ((a.w_bytes + 1023u) & ~1023u);
  const uint32_t off_stg = ((a.w_bytes + 1023u) & ~1023u) + S * halo_bytes;
  const uint32_t off_bar = off_stg + H_STAGING_BYTES;
  const uint32_t bars = base + off_bar;
  // barriers: w_full, halo_full[S], halo_empty[S]
  const uint32_t w_full = bars;
  auto halo_full = [&](int s) { return bars + 8u * (1 + s); };
  auto halo_empty = [&](int s) { return bars + 8u * (1 + S + s); };

  pdl_trigger();                       // the next kernel of the stream may start its own prologue now
  if (tid == 0) {
    mbar_init(w_full, 1);
    // a halo stage is read by both warpgroups, or (pixel-major) by the one whose item it holds
    for (int s = 0; s < S; ++s) { mbar_init(halo_full(s), 1); mbar_init(halo_empty(s), PX::on ? 4 : H_MMA_WARPS); }
    mbar_init_fence();
  }
  // folded-BN shift / bias of this CTA's output-channel tile, staged once (read as float4 broadcasts)
  float* s_shift = reinterpret_cast<float*>(sm + off_bar + 256);      // barriers use <= 136 bytes at S = 8
  {
    const int n0s = (blockIdx.x % a.n_tiles_n) * N;
    for (int j = tid; j < 256; j += H_THREADS)
      s_shift[j] = (a.shift && j < N && n0s + j < g.C_out) ? __ldg(a.shift + n0s + j) : 0.f;
  }
  __syncthreads();
  // the weights are constants: their bulk copy goes out BEFORE waiting for the previous kernel (PDL), so that it
  // overlaps that kernel's tail; everything after the wait reads activations the previous kernel produced
  if (warp == 8 && lane == 0) {
    mbar_arrive_expect_tx(w_full, a.w_bytes);
    bulk_g2s(sW, reinterpret_cast<const unsigned char*>(a.w) + (size_t)(blockIdx.x % a.n_tiles_n) * a.w_bytes, a.w_bytes, w_full);
  }
  pdl_wait();

  // work items: n-tile major so that a CTA keeps ONE weight tile resident:  item = nt * spatial + sp
  // CTA c handles n-tile (c % n_tiles_n) and spatial tiles (c / n_tiles_n) + i * (gridDim.x / n_tiles_n)
  const int nt = blockIdx.x % a.n_tiles_n;
  const int sp0 = blockIdx.x / a.n_tiles_n;
  const int sp_stride = gridDim.x / a.n_tiles_n;
  const int sp_total = a.tiles_total;
  const int n0 = nt * N;
  const int per_img = a.tiles_x * a.tiles_y;

  if (warp == 8) {
    if (lane == 0) {
      // ===================== TMA producer =====================
      int it = 0;
      for (int sp = sp0; sp < sp_total; sp += sp_stride, ++it) {
        const int s = it % S;
        const uint32_t ph = (uint32_t)(it / S) & 1u;
        mbar_wait(halo_empty(s), ph ^ 1u, 1, it);
        h_stamp(trace, it, 0);
        const int b = sp / per_img, r = sp - b * per_img;
        const int ty = r / a.tiles_x, tx = r - ty * a.tiles_x;
        const int x0 = tx * a.tw - g.pad, y0 = ty * a.th - g.pad;
        mbar_arrive_expect_tx(halo_full(s), (uint32_t)(a.planes * a.box_bytes));   // TMA writes the full box (zero fill incl.)
        if (a.merged_xc) {
          tma_3d(sH + s * halo_bytes, &tmap, x0 * 8, y0, b, halo_full(s));
        } else {
          // un-swizzled: one 8-channel plane per copy; swizzled: one <=64-channel chunk (whole 128-byte rows)
          const int cstep = a.swz ? (a.swz >> 1) : 8;
          for (int p = 0; p < a.planes; ++p)
            tma_4d(sH + s * halo_bytes + p * a.plane_bytes, &tmap, p * cstep, x0, y0, b, halo_full(s));
        }
        h_stamp(trace, it, 1);
      }
    }
  } else if constexpr (PX::on) {
    // ===================== pixel-major MMA + epilogue warpgroups (see the top of the file) =====================
    const int wg = warp >> 2, w4 = warp & 3;
    const bool lead = (tid & 127) == 0;          // stamps the trace of this warpgroup's items
    const uint32_t stg = base + off_stg + (uint32_t)wg * (64u * EPI_PITCH * 4u);
    // A (weights, K-major no-swizzle): LBO = next 8 k (64 x 16 B), SBO = next 8 channels (128 B); 64 x 32 B per block
    const uint64_t w_desc0 = wg_desc(sW, 64u * 16u, 128u, 0u);
    const uint64_t h_hi = (uint64_t)a.m_ahi << 32;
    // epilogue pass j (pixels 32j .. 32j + 31 of the item): thread = pixel 32j + lane, channels 16 w4 .. 16 w4 + 15
    const int gy = lane >> 3, rx = lane & 7;     // pixel 32j + lane = (tile row 4j + gy, x rx)
    // passes whose residual is prefetched (2 x 16 B of registers each): all four under the one-CTA register cap, none
    // under the two-CTA one (the accumulator alone is 64 registers)
    constexpr int PF = OVERLAP ? 4 : 0;
    uint4 rq[PF > 0 ? PF : 1][2];
    const bool use_res = a.residual != nullptr;
    auto prefetch_residual = [&](int sp_n) {
      const int bn = sp_n / per_img, rn = sp_n - bn * per_img;
      const int tyn = rn / a.tiles_x, txn = rn - tyn * a.tiles_x;
      const int oxn = txn * HT_W + rx;
#pragma unroll
      for (int j = 0; j < PF; ++j) {
        const int oyn = tyn * HT_H + 4 * j + gy;
        rq[j][0] = make_uint4(0, 0, 0, 0); rq[j][1] = make_uint4(0, 0, 0, 0);
        if (oyn < g.OH && oxn < g.OW) {
          const uint4* rp = reinterpret_cast<const uint4*>(
              a.residual + (((size_t)bn * g.OH + oyn) * g.OW + oxn) * g.ld_res + 16 * w4);
          rq[j][0] = __ldg(rp); rq[j][1] = __ldg(rp + 1);
        }
      }
    };
    const int sp_first = sp0 + wg * sp_stride, sp_step = 2 * sp_stride;
    if (PF > 0 && use_res && sp_first < sp_total) prefetch_residual(sp_first);
    // folded-BN shifts of this thread's two accumulator rows (channels 16 w4 + lane / 4, + 8)
    const float sh0 = s_shift[16 * w4 + (lane >> 2)], sh1 = s_shift[16 * w4 + (lane >> 2) + 8];
    mbar_wait(w_full, 0, 2, 0);
    // OVERLAP: the chains take turns in item order (warpgroup 0's item 0, warpgroup 1's item 1, ...), on the named
    // barriers of the other flavour; after the loop the warpgroup that did not run the last item consumes the last
    // arrival.
    const int n_items = sp0 < sp_total ? (sp_total - sp0 - 1) / sp_stride + 1 : 0;
    if constexpr (OVERLAP)
      if (wg == 1 && n_items > 0) named_arrive(3, 256);
    float acc[64];
    int it = wg;
    for (int sp = sp_first; sp < sp_total; sp += sp_step, it += 2) {
      const int s = it % S;
      const uint32_t ph = (uint32_t)(it / S) & 1u;
      if constexpr (OVERLAP) named_sync(3 + wg, 256);
      mbar_wait(halo_full(s), ph, 3, it);
      if (lead) h_stamp(trace, it, 2);
      const uint32_t h_lo0 = a.m_alo + (sH >> 4) + ((uint32_t)s * halo_bytes >> 4);
      wg_fence();
#pragma unroll
      for (int ky = 0; ky < PX::ky; ++ky)
#pragma unroll
        for (int kx = 0; kx < PX::kx; ++kx)
#pragma unroll
          for (int c = 0; c < PX::nc; ++c)
#pragma unroll
            for (int qq = 0; qq < PX::nq; ++qq) {
              const int blk = ((ky * PX::kx + kx) * PX::nc + c) * PX::nq + qq;
              const uint32_t h_lo = h_lo0 + (uint32_t)ky * a.m_sky + (uint32_t)kx * a.m_skx + (uint32_t)c * a.m_sc +
                                    (uint32_t)qq * a.m_sq;
              Wgmma<128>::mma(acc, w_desc0 + (uint64_t)(blk * 128), h_hi | h_lo, blk > 0 ? 1u : 0u);
            }
      wg_commit();
      wg_wait<0>();
      wg_fence_operand(acc);
      if constexpr (OVERLAP) named_arrive(3 + (wg ^ 1), 256);
      __syncwarp();
      if (lane == 0) mbar_arrive(halo_empty(s));     // this warp's MMAs no longer read the halo stage
      if (lead) h_stamp(trace, it, 4);

      // ---- epilogue: acc[4 i + 2 h + e] = channel 16 w4 + lane / 4 + 8 h, pixel 8 i + 2 (lane % 4) + e
      const int b = sp / per_img, r = sp - b * per_img;
      const int ty = r / a.tiles_x, tx = r - ty * a.tiles_x;
      const int ox = tx * HT_W + rx;
      if (lead) h_stamp(trace, it, 5);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        named_sync(1 + wg, 128);                   // the previous pass's readers are done with the staging tile
        // + shift, transposed into the staging tile [32 pixels][PX_PITCH]
#pragma unroll
        for (int i = 4 * j; i < 4 * j + 4; ++i)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const uint32_t px = (uint32_t)(8 * (i - 4 * j) + 2 * (lane & 3) + e);
              const uint32_t ch = (uint32_t)(16 * w4 + (lane >> 2) + 8 * h);
              const float v = acc[4 * i + 2 * h + e] + (h ? sh1 : sh0);
              sts32(stg + (px * PX_PITCH + ch) * 4u, __float_as_uint(v));
            }
        named_sync(1 + wg, 128);
        const int oy = ty * HT_H + 4 * j + gy;
        if (oy >= g.OH || ox >= g.OW) continue;
        const size_t p = a.out_s2d ? ((((size_t)b * (g.OH >> 1) + (oy >> 1)) * (g.OW >> 1) + (ox >> 1)) << 2) + (((oy & 1) << 1) | (ox & 1))
                                   : ((size_t)b * g.OH + oy) * g.OW + ox;
        float v[16];
        lds_f(stg + ((uint32_t)lane * PX_PITCH + 16u * w4) * 4u, v);
        if (use_res) {
          uint4 ra, rb;
          if (j < PF) {
            ra = rq[j < PF ? j : 0][0]; rb = rq[j < PF ? j : 0][1];
          } else {
            const uint4* rp = reinterpret_cast<const uint4*>(a.residual + p * g.ld_res + 16 * w4);
            ra = __ldg(rp); rb = __ldg(rp + 1);
          }
          add_residual_bf16(v, ra, rb);
        }
        relu16(v, g.relu);
        store_bf16x16(reinterpret_cast<__nv_bfloat16*>(a.out) + p * g.ld_out + 16 * w4, v);
      }
      if (PF > 0 && use_res && sp + sp_step < sp_total) prefetch_residual(sp + sp_step);
      if (lead) h_stamp(trace, it, 6);
    }
    if constexpr (OVERLAP)
      if (n_items > 0 && wg != ((n_items - 1) & 1)) named_sync(3 + wg, 256);
  } else {
    // ===================== MMA + epilogue warpgroups =====================
    const int wg = warp >> 2, w4 = warp & 3;
    const int lrow = 32 * (w4 & 1) + lane;       // row of this warpgroup's 64 (epilogue: row per thread)
    const int chalf = w4 >> 1;                   // 16-column half of each 32-column chunk
    const int row = 64 * wg + lrow;              // GEMM row = g*8 + r  ->  pixel (ty*16 + g, tx*8 + r)
    const uint32_t stg = base + off_stg + (uint32_t)wg * (64u * EPI_PITCH * 4u);
    // B (weights, K-major no-swizzle): core matrices of 8 channels x 16 B, LBO = next 8 k (n_tile x 16 B), SBO = 128 B
    const uint64_t b_desc0 = wg_desc(sW, (uint32_t)N * 16u, 128u, 0u);
    const uint32_t b_step = ((uint32_t)N * 32u) >> 4;               // descriptor start-address units (16 B) per block
    // this warpgroup's m64 half starts 8 core-matrix groups (8 x SBO) into the tile
    const uint32_t half16 = (uint32_t)wg * 8u * (a.m_ahi & 0x3FFFu);
    // 8 consecutive GEMM rows = 8 consecutive x; the 8-row groups then run along x (tw / 8 of them) before y
    const int gpr = a.tw >> 3;
    const int gy = (row >> 3) / gpr, rx = (((row >> 3) % gpr) << 3) | (row & 7);
    const int HWo = g.OH * g.OW;
    // Residual tiles are prefetched one work item ahead into registers (the load does not depend on the MMA):
    // issued right after the previous item consumed its copy, they land while this warp runs the next item's MMAs.
    constexpr int PF = 2;                      // 16-column chunks per thread that can be prefetched (n_tile <= 64)
    uint4 rq[PF][2];
    const bool use_res = a.residual != nullptr && g.out_mode == CT_OUT_NHWC && !a.sum3;
    auto prefetch_residual = [&](int sp_n) {
      const int bn = sp_n / per_img, rn = sp_n - bn * per_img;
      const int tyn = rn / a.tiles_x, txn = rn - tyn * a.tiles_x;
      const int oyn = tyn * a.th + gy, oxn = txn * a.tw + rx;
      const bool okn = oyn < g.OH && oxn < g.OW;
      const size_t pn = ((size_t)bn * g.OH + oyn) * g.OW + oxn;
#pragma unroll
      for (int i = 0; i < PF; ++i) {
        const int col = chalf * 16 + 32 * i;
        rq[i][0] = make_uint4(0, 0, 0, 0); rq[i][1] = make_uint4(0, 0, 0, 0);
        if (okn && col < N && n0 + col < g.C_out) {
          const uint4* rp = reinterpret_cast<const uint4*>(a.residual + pn * g.ld_res + n0 + col);
          rq[i][0] = __ldg(rp); rq[i][1] = __ldg(rp + 1);
        }
      }
    };
    if (use_res && sp0 < sp_total) prefetch_residual(sp0);
    mbar_wait(w_full, 0, 2, 0);
    // OVERLAP (ping-pong): the two warpgroups' chains take turns on the tensor cores -- warpgroup 0's chain of item it,
    // then warpgroup 1's, then warpgroup 0's of item it + 1 -- so each warpgroup's epilogue runs while the other's MMAs
    // do.  Named barrier 3 + w: "warpgroup w may issue", arrived on by the other warpgroup once its chain is complete
    // (warpgroup 1 also arrives once up front, for warpgroup 0's first chain, and warpgroup 0 consumes its last
    // arrival after the loop).  The barrier calls in the loop are unconditional: a branch next to the MMAs would make
    // ptxas serialise them.
    if constexpr (OVERLAP)
      if (wg == 1 && sp0 < sp_total) named_arrive(3, 256);
    float acc[N / 2];
    int it = 0;
    for (int sp = sp0; sp < sp_total; sp += sp_stride, ++it) {
      const int s = it % S;
      const uint32_t ph = (uint32_t)(it / S) & 1u;
      if constexpr (OVERLAP) named_sync(3 + wg, 256);
      mbar_wait(halo_full(s), ph, 3, it);
      if (tid == 0) h_stamp(trace, it, 2);
      // A-descriptor walk (ky, kx|pair, chunk, K-step): warp-uniform adds on the start address; B advances by b_step
      const uint32_t a_lo0 = a.m_alo + (sH >> 4) + ((uint32_t)s * halo_bytes >> 4) + half16;
      uint64_t b_desc = b_desc0;
      uint32_t accum = 0;
      wg_fence();
      for (int ky = 0; ky < a.m_nky; ++ky)
        for (int kx = 0; kx < a.m_nkx; ++kx)
          for (int c = 0; c < a.m_nc; ++c)
            for (int qq = 0; qq < a.m_nq; ++qq) {
              const uint32_t a_lo = a_lo0 + (uint32_t)ky * a.m_sky + (uint32_t)kx * a.m_skx + (uint32_t)c * a.m_sc +
                                    (uint32_t)qq * a.m_sq;
              Wgmma<N>::mma(acc, ((uint64_t)a.m_ahi << 32) | (uint64_t)a_lo, b_desc, accum);
              accum = 1;
              b_desc += b_step;
            }
      wg_commit();
      wg_wait<0>();
      wg_fence_operand(acc);
      if constexpr (OVERLAP) named_arrive(3 + (wg ^ 1), 256);
      __syncwarp();
      if (lane == 0) mbar_arrive(halo_empty(s));     // this warp's MMAs no longer read the halo stage
      if (tid == 0) h_stamp(trace, it, 4);

      // ---- epilogue of this warpgroup's 64 rows
      const int b = sp / per_img, r = sp - b * per_img;
      const int ty = r / a.tiles_x, tx = r - ty * a.tiles_x;
      const int oy = ty * a.th + gy, ox = tx * a.tw + rx;
      const bool p_ok = oy < g.OH && ox < g.OW;
      const size_t p = a.out_s2d ? ((((size_t)b * (g.OH >> 1) + (oy >> 1)) * (g.OW >> 1) + (ox >> 1)) << 2) + (((oy & 1) << 1) | (ox & 1))
                                 : ((size_t)b * g.OH + oy) * g.OW + ox;
      if (tid == 0) h_stamp(trace, it, 5);
      float s8[8];                                   // stem (sum3) partial sums, carried across the chunks
#pragma unroll
      for (int j = 0; j < 8; ++j) s8[j] = 0.f;
#pragma unroll
      for (int c0 = 0; c0 < N; c0 += 32) {
        named_sync(1 + wg, 128);                   // the previous chunk's readers are done with the staging tile
        stage_acc_chunk(acc, c0, stg, 0);
        named_sync(1 + wg, 128);
        const uint32_t srow = stg + (uint32_t)lrow * EPI_PITCH * 4u;
        if (a.sum3) {
          // stem: three 16-channel groups, ReLU each (after its folded-BN shift), then sum (dla.py:307-311).
          // Warp half `chalf` produces output channels 8*chalf .. 8*chalf+7 (columns g*16 + 8*chalf + j).
#pragma unroll
          for (int grp = 0; grp < 3; ++grp) {
            if (grp * 16 < c0 || grp * 16 >= c0 + 32 || grp * 16 >= N) continue;
            if (!((a.sum3 >> grp) & 1)) continue;          // absent input (pre_img / pre_hm is None)
            float rr[8];
            lds_f(srow + (uint32_t)(grp * 16 - c0 + chalf * 8) * 4u, rr);
            const float4* sh4 = reinterpret_cast<const float4*>(s_shift + grp * 16 + chalf * 8);
            const float4 sa = sh4[0], sb = sh4[1];
            s8[0] += fmaxf(rr[0] + sa.x, 0.f); s8[1] += fmaxf(rr[1] + sa.y, 0.f);
            s8[2] += fmaxf(rr[2] + sa.z, 0.f); s8[3] += fmaxf(rr[3] + sa.w, 0.f);
            s8[4] += fmaxf(rr[4] + sb.x, 0.f); s8[5] += fmaxf(rr[5] + sb.y, 0.f);
            s8[6] += fmaxf(rr[6] + sb.z, 0.f); s8[7] += fmaxf(rr[7] + sb.w, 0.f);
          }
          continue;
        }
        const int col = c0 + chalf * 16;
        const int o0 = n0 + col;
        if (col >= N || !p_ok || o0 >= g.C_out) continue;
        float v[16];
        lds_f(srow + (uint32_t)chalf * 64u, v);
        const float4* sh4 = reinterpret_cast<const float4*>(s_shift + col);
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) {
          const float4 sh = sh4[j4];
          v[4 * j4 + 0] += sh.x; v[4 * j4 + 1] += sh.y; v[4 * j4 + 2] += sh.z; v[4 * j4 + 3] += sh.w;
        }
        if (g.out_mode == CT_OUT_NHWC) {
          if (a.residual) {
            uint4 ra, rb;
            const int ci = col >> 5;                     // this thread's chunk index
            if (ci < PF) {
              ra = rq[0][0]; rb = rq[0][1];
#pragma unroll
              for (int i = 1; i < PF; ++i) if (ci == i) { ra = rq[i][0]; rb = rq[i][1]; }
            } else {
              const uint4* rp = reinterpret_cast<const uint4*>(a.residual + p * g.ld_res + o0);
              ra = __ldg(rp); rb = __ldg(rp + 1);
            }
            add_residual_bf16(v, ra, rb);
          }
          relu16(v, g.relu);
          store_bf16x16(reinterpret_cast<__nv_bfloat16*>(a.out) + p * g.ld_out + o0, v);
        } else if (g.out_mode == CT_OUT_NHWC_F32) {
          store_f32_nhwc16(reinterpret_cast<float*>(a.out) + p * g.ld_out + o0, v, o0, g);
        } else {
          store_head16(reinterpret_cast<float*>(a.out) + ((size_t)b * g.C_out + o0) * HWo + (size_t)oy * g.OW + ox, HWo,
                       v, o0, g);
        }
      }
      if (a.sum3 && p_ok) {
        uint4 o;
        __nv_bfloat162* po = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
        for (int j = 0; j < 4; ++j) po[j] = __floats2bfloat162_rn(s8[2 * j], s8[2 * j + 1]);
        *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(a.out) + p * g.ld_out + chalf * 8) = o;
      }
      if (use_res && sp + sp_stride < sp_total) prefetch_residual(sp + sp_stride);
      if (tid == 0) h_stamp(trace, it, 6);
    }
    if constexpr (OVERLAP)
      if (wg == 0 && sp0 < sp_total) named_sync(3, 256);
  }
}

// ---- host ----
int halo_set_trace(void* buf) {
  unsigned long long* p = (unsigned long long*)buf;
  return cudaMemcpyToSymbol(g_halo_trace, &p, sizeof(p)) == cudaSuccess ? CT_OK : CT_ERR_CUDA;
}
int halo_set_watch(void* mapped_host_buf) { return set_mbar_watch(mapped_host_buf); }

int halo_blocks(int C_in, int KH, int KW) {
  return C_in == 8 ? KH * ((KW + 1) / 2) : KH * KW * (C_in / 16);
}

// Configuration step: the launch arguments other than the pointers, and the launch configuration.  No CUDA call.
static int halo_config(const ct_conv_desc* d, HaloArgs& a, ConvConfig& c) {
  a.g = make_geom(d);
  const ConvGeom& g = a.g;
  if (g.stride != 1 || g.pad != g.KH / 2 || g.KH != g.KW || g.OH != g.H || g.OW != g.W)
    return fail(CT_ERR_INVALID, "conv_halo: stride-1 'same' convolutions only%s", "");
  if (!(g.C_in == 8 || (g.C_in % 16 == 0 && g.C_in <= 64) || (g.C_in % 64 == 0 && g.C_in <= 256)) || g.ld_in % 8 != 0)
    return fail(CT_ERR_INVALID, "conv_halo: C_in must be 8, 16, 32, 48, 64, 128, 192 or 256 (ld_in %% 8 == 0)%s (%ld)", "", g.C_in);
  const int n_tile = d->n_tile;
  if (n_tile <= 0 || n_tile % 16 != 0 || n_tile > 256)
    return fail(CT_ERR_INVALID, "conv_halo: bad n_tile%s (%ld)", "", n_tile);
  a.sum3 = d->epilogue_sum3;
  a.out_s2d = 0;
  if (g.out_mode == CT_OUT_NHWC_S2D) {
    if ((g.OH | g.OW) & 1 || d->residual)
      return fail(CT_ERR_INVALID, "conv_halo: CT_OUT_NHWC_S2D needs even OH / OW, no residual%s", "");
    a.out_s2d = 1;
    a.g.out_mode = CT_OUT_NHWC;
  }
  if (a.sum3 && !(g.C_out == 48 && n_tile == 48 && g.out_mode == CT_OUT_NHWC && d->shift))
    return fail(CT_ERR_INVALID, "conv_halo: sum3 epilogue needs C_out == n_tile == 48, NHWC output, shift%s", "");
  if (g.out_mode == CT_OUT_NHWC && !a.sum3 && (g.C_out % 16 != 0 || g.ld_out % 8 != 0))
    return fail(CT_ERR_INVALID, "conv_halo: NHWC bf16 output needs C_out %% 16 == 0, ld_out %% 8 == 0%s", "");
  if (d->residual && (g.out_mode != CT_OUT_NHWC || g.ld_res % 8 != 0))
    return fail(CT_ERR_INVALID, "conv_halo: residual only for NHWC bf16 outputs, ld_res %% 8 == 0%s", "");
  a.n_tile = n_tile;
  a.n_tiles_n = (g.C_out + n_tile - 1) / n_tile;
  a.pair_taps = g.C_in == 8;
  a.nblk = halo_blocks(g.C_in, g.KH, g.KW);
  if (a.nblk > 160) return fail(CT_ERR_UNSUPPORTED, "conv_halo: more than 160 K=16 blocks per tile%s (%ld)", "", (long)a.nblk);
  // operand staging mode: whole-pixel swizzled rows when C_in*2 is a swizzle width (one 32/64/128-byte TMA
  // request per halo pixel); C_in == 8 keeps the 16-byte un-swizzled rows but merges (x, c) in the tensor map
  // when the tensor is dense (ld_in == 8) so that one request covers a whole halo row.
  static const bool force_planes = [] { const char* e = getenv("CTB_HALO_MODE"); return e && strcmp(e, "planes") == 0; }();   // debug
  a.swz = (g.C_in > 64) ? 128 : ((!force_planes && (g.C_in == 16 || g.C_in == 32 || g.C_in == 64)) ? g.C_in * 2 : 0);
  a.merged_xc = (g.C_in == 8 && g.ld_in == 8) ? 1 : 0;
  a.planes = a.swz ? (g.C_in * 2 + a.swz - 1) / a.swz : g.C_in / 8;   // swizzled: 64-channel chunks
  // 1x1 convs writing fp32 NCHW planes (the 1x1 heads) use a 32 x 4 pixel tile: there is no halo, the TMA box
  // [4][32][c] is already the canonical K-major operand (8-pixel groups 8 rows apart), and every epilogue warp then
  // owns 32 consecutive x of one row: its per-channel store is one full 128-byte line instead of four 32-byte pieces.
  a.tw = HT_W; a.th = HT_H;
  static const int wide_env = getenv("CTB_HALO_WIDE") ? atoi(getenv("CTB_HALO_WIDE")) : 1;
  if (wide_env && g.KH == 1 && g.KW == 1 && g.out_mode == CT_OUT_NCHW_F32 && a.swz && g.OW % 32 == 0 && g.OH % 4 == 0) {
    a.tw = 32; a.th = 4;
  }
  a.pw = a.tw + g.KW - 1 + (a.pair_taps ? 1 : 0);
  a.ph = a.th + g.KH - 1;
  a.box_bytes = a.pw * a.ph * (a.swz ? a.swz : 16);
  a.plane_bytes = (a.box_bytes + 1023) / 1024 * 1024;
  a.w_bytes = (uint32_t)a.nblk * n_tile * 32u;
  if (a.pair_taps) {                 // one MMA = taps (ky, 2kp) and (ky, 2kp+1): K-core 1 is the next pixel
    a.m_nky = g.KH; a.m_nkx = (g.KW + 1) / 2; a.m_nc = 1; a.m_nq = 1;
    a.m_sky = a.pw; a.m_skx = 2; a.m_sc = 0; a.m_sq = 0;
    a.m_alo = 1u << 16;                                   // LBO = 16 B
    a.m_ahi = (uint32_t)a.pw;                             // SBO = pw*16 B
  } else if (a.swz) {
    const uint32_t rb16 = (uint32_t)a.swz >> 4;
    a.m_nky = g.KH; a.m_nkx = g.KW; a.m_nc = a.planes; a.m_nq = (g.C_in < 64 ? g.C_in : 64) / 16;
    a.m_sky = (uint32_t)a.pw * rb16; a.m_skx = rb16; a.m_sc = (uint32_t)a.plane_bytes >> 4; a.m_sq = 2;
    a.m_alo = 1u << 16;
    const uint32_t layout = a.swz == 128 ? 1u : (a.swz == 64 ? 2u : 3u);      // descriptor bits [62,64)
    const uint32_t sbo16 = a.tw == HT_W ? (uint32_t)a.pw * rb16 : 8u * rb16;     // next 8-row group: next tile row / next 8 px
    a.m_ahi = sbo16 | (layout << 30);
  } else {
    a.m_nky = g.KH; a.m_nkx = g.KW; a.m_nc = 1; a.m_nq = g.C_in / 16;
    a.m_sky = a.pw; a.m_skx = 1; a.m_sc = 0; a.m_sq = 2u * ((uint32_t)a.plane_bytes >> 4);
    a.m_alo = ((uint32_t)a.plane_bytes >> 4) << 16;       // LBO = plane stride
    a.m_ahi = (uint32_t)a.pw;
  }
  // pixel-major: the 64 -> 64-channel layers with NHWC bf16 output, for the walks PX_WALKS instantiates
  a.px = 0;
  if (n_tile == 64 && g.C_out == 64 && g.out_mode == CT_OUT_NHWC && !a.sum3 && a.swz && !a.pair_taps && a.tw == HT_W)
    for (int i = 0; i < (int)(sizeof(PX_WALKS) / sizeof(PX_WALKS[0])); ++i)
      if (g.KH == PX_WALKS[i][0] && g.KW == PX_WALKS[i][1] && g.C_in == PX_WALKS[i][2]) a.px = i + 1;
  a.tiles_x = (g.OW + a.tw - 1) / a.tw;
  a.tiles_y = (g.OH + a.th - 1) / a.th;
  a.tiles_total = g.B * a.tiles_x * a.tiles_y;
  const size_t halo_bytes = (size_t)a.planes * a.plane_bytes;
  auto smem_for = [&](int s) { return (size_t)((a.w_bytes + 1023) & ~1023u) + s * halo_bytes + H_STAGING_BYTES + 256 + 1024 + 1024; };
  auto ctas_for = [&](int s) {
    const int n = (int)((227 * 1024) / smem_for(s));
    return n > 2 ? 2 : n;                 // register file: 2 x 288 threads x <= 112 registers
  };
  // Halo stages: as many (up to 4) as keep the CTAs-per-SM count -- the TMA of a thin-channel halo (32-byte rows)
  // lands thousands of cycles after it is issued, so one stage in flight would leave the MMAs waiting.
  int stages = 2;
  for (int sdeep = 4; sdeep >= 3; --sdeep)
    if (smem_for(sdeep) <= 227 * 1024 && ctas_for(sdeep) == ctas_for(2)) { stages = sdeep; break; }
  static const int stages_env = getenv("CTB_HALO_STAGES") ? atoi(getenv("CTB_HALO_STAGES")) : 0;
  if (stages_env >= 2) stages = stages_env;
  if (smem_for(stages) > 227 * 1024)
    return fail(CT_ERR_UNSUPPORTED, "conv_halo: weights + halo do not fit in shared memory%s (%ld bytes)", "",
                (long)smem_for(stages));
  a.halo_stages = stages;
  // the persistent grid is sized for this many CTAs per SM
  int per_sm = ctas_for(stages);
  if (n_tile > 128) per_sm = 1;     // wide tiles: one CTA per SM (accumulator registers)
  // One CTA per SM: no second CTA's MMAs fill this one's epilogue, so its two warpgroups take turns (overlap).  Not
  // below N = 64: one warpgroup's m64n32 chain alone is bound by its shared-memory operand reads and leaves the tensor
  // pipe half idle, so the two chains must run together (measured: the 128 -> 128 N = 32 layers 45 % slower in turns).
  // CTB_HALO_OVERLAP=0: the serial schedule everywhere, for A/B runs; the outputs are bit-identical.
  static const int overlap_env = getenv("CTB_HALO_OVERLAP") ? atoi(getenv("CTB_HALO_OVERLAP")) : 1;
  c.smem_bytes = (int32_t)smem_for(stages);
  c.stages = stages;
  c.tile_w = a.tw;
  c.tile_h = a.th;
  c.ctas_per_sm = per_sm;
  c.overlap = overlap_env && per_sm == 1 && n_tile >= 64 && n_tile <= 128;
  c.pixel_major = a.px != 0;
  return CT_OK;
}

int conv_config_halo(const ct_conv_desc* d, ConvConfig* c) {
  HaloArgs a;
  return halo_config(d, a, *c);
}

int conv_forward_halo(const ct_conv_desc* d, cudaStream_t st) {
  HaloArgs a;
  ConvConfig c;
  const int rc = halo_config(d, a, c);
  if (rc != CT_OK) return rc;
  if (((uintptr_t)d->x & 15) || ((uintptr_t)d->w & 15) || ((uintptr_t)d->out & 15) || ((uintptr_t)d->residual & 15))
    return fail(CT_ERR_INVALID, "conv_halo: x/w/out/residual must be 16-byte aligned%s", "");
  a.w = (const __nv_bfloat16*)d->w;
  a.shift = d->shift;
  a.residual = (const __nv_bfloat16*)d->residual;
  a.out = d->out;
  const ConvGeom& g = a.g;

  CUtensorMap tmap;
  int r;
  if (a.merged_xc) {
    const cuuint64_t dims[3] = {(cuuint64_t)g.W * 8, (cuuint64_t)g.H, (cuuint64_t)g.B};
    const cuuint64_t strides[2] = {(cuuint64_t)g.W * 16, (cuuint64_t)g.H * g.W * 16};
    const cuuint32_t box[3] = {(cuuint32_t)a.pw * 8, (cuuint32_t)a.ph, 1};
    r = encode_tmap_bf16(&tmap, d->x, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE);
  } else {
    const cuuint64_t dims[4] = {(cuuint64_t)g.C_in, (cuuint64_t)g.W, (cuuint64_t)g.H, (cuuint64_t)g.B};
    const cuuint64_t strides[3] = {(cuuint64_t)g.ld_in * 2, (cuuint64_t)g.W * g.ld_in * 2,
                                   (cuuint64_t)g.H * g.W * g.ld_in * 2};
    const cuuint32_t box[4] = {(cuuint32_t)(a.swz ? a.swz / 2 : 8), (cuuint32_t)a.pw, (cuuint32_t)a.ph, 1};
    const CUtensorMapSwizzle sw = a.swz == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                  : a.swz == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                  : a.swz == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE;
    r = encode_tmap_bf16(&tmap, d->x, 4, dims, strides, box, sw);
  }
  if (r != CT_OK) return r;

  // persistent grid: a multiple of n_tiles_n, at most (SMs x CTAs that fit) and no more than the work
  const int sms = device_sm_count();
  long want = (long)sms * c.ctas_per_sm;
  long groups = want / a.n_tiles_n;
  if (groups < 1) groups = 1;
  if (groups > a.tiles_total) groups = a.tiles_total;
  const int grid = (int)(groups * a.n_tiles_n);
  if (a.px) {
    auto launch_px = [&](auto px) {
      using PX = decltype(px);
      if (a.m_nky != PX::ky || a.m_nkx != PX::kx || a.m_nc != PX::nc || a.m_nq != PX::nq)
        return fail(CT_ERR_INVALID, "conv_halo: pixel-major walk does not match the layer%s", "");
      return c.overlap ? launch_big_smem<conv_halo_kernel<64, true, PX>>(dim3(grid), dim3(H_THREADS), c.smem_bytes, st, a, tmap)
                       : launch_big_smem<conv_halo_kernel<64, false, PX>>(dim3(grid), dim3(H_THREADS), c.smem_bytes, st, a, tmap);
    };
    static_assert(sizeof(PX_WALKS) / sizeof(PX_WALKS[0]) == 4, "one case per walk");
    switch (a.px) {
      case 1: return launch_px(PxWalk<3, 3, 1, 4>{});
      case 2: return launch_px(PxWalk<2, 2, 2, 4>{});
      case 3: return launch_px(PxWalk<1, 1, 1, 2>{});
      default: return launch_px(PxWalk<1, 1, 2, 4>{});
    }
  }
  return dispatch_n_tile(a.n_tile, [&](auto n) {
    constexpr int NT = decltype(n)::value;
    if constexpr (NT >= 64 && NT <= 128)
      if (c.overlap)
        return launch_big_smem<conv_halo_kernel<NT, true>>(dim3(grid), dim3(H_THREADS), c.smem_bytes, st, a, tmap);
    return launch_big_smem<conv_halo_kernel<NT, false>>(dim3(grid), dim3(H_THREADS), c.smem_bytes, st, a, tmap);
  });
}

}  // namespace ctb
