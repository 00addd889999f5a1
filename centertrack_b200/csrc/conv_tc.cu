// wgmma implicit-GEMM convolution / DCNv2 for sm_90a (bf16 operands, fp32 accumulate in registers).
//
//   D[128 pixels x n_tile channels]  +=  A[128 x 64] (smem, gathered)  x  B[n_tile x 64]^T (smem)
//
// * No im2row buffer in HBM: each warpgroup gathers its 64 rows of every 64-wide K slice (tap-major,
//   k = tap*C_in + c) of the A operand straight into the 128B-swizzled K-major shared-memory layout the
//   wgmma descriptor expects.  For CT_A_DCN the gather is the DCNv2 bilinear sample x mask (the reference's
//   `columns` tensor never exists).
// * Weights are pre-packed on the host as ready-made swizzled tile images, so one TMA bulk copy
//   (cp.async.bulk, mbarrier complete_tx) per K slice brings the B tile.
// * CTA = 256 threads = two warpgroups.  Warpgroup w gathers rows 64w..64w+63 and issues wgmma
//   (M=64, N=n_tile, K=16) x4 per slice on them; the MMAs of slice s run while the warpgroup gathers slice s+1
//   (wgmma.wait_group 1), and one arrival per warp on the stage's empty barrier releases the weight tile.
// * Epilogue: the register accumulator goes through shared memory 32 columns at a time (row per thread), then
//   + folded-BN shift, + residual, ReLU, bf16 NHWC / fp32 NHWC (DCN offsets, sigmoid on the mask channels) /
//   fp32 NCHW (heads, sigmoid / depth transform) stores.
#include "conv_common.cuh"
#include "wgmma.cuh"
#include <cuda.h>
#include <stdlib.h>

namespace ctb {

constexpr int TC_BM = 128;           // output pixels per CTA
constexpr int TC_BK = 64;            // K elements per pipeline stage (one 128B swizzle atom of bf16)
constexpr int TC_THREADS = 256;      // two warpgroups: gather + MMA + epilogue
constexpr int TC_PRODUCERS = 256;
constexpr int TC_NROW = TC_BM * 8 / TC_PRODUCERS;   // A-tile rows per thread per K slice (4, 16 rows apart)
constexpr int A_STAGE_BYTES = TC_BM * 128;

struct TcArgs {
  ConvGeom g;
  const __nv_bfloat16* x;       // X3 engine: fp32 activations behind the same pointers (xf() / residual_f())
  const __nv_bfloat16* w;       // packed tiles (X3: [hi tile][lo tile] per K slice)
  const float* shift;
  const __nv_bfloat16* residual;
  const float* om;
  void* out;
  int n_tile, k_slices, stages, a_mode;
  int tiles_x, tiles_y;         // > 0: an M tile is an 8 (y) x 16 (x) pixel patch of one image (L1 reuse of the
                                // 3x3 / bilinear footprints); 0: 128 consecutive pixels in b,y,x order
  int win_m, win_pw, win_ph;    // CT_A_DCN_WIN: offset margin (px) and the staged window (pixels) of one 8x16 patch
  uint32_t win_bytes;           // bytes of one 64-channel window (= TMA box)
  uint32_t region0;             // bytes of the stage area (also holds the epilogue staging tile)
};

// CT_A_DCN_WIN sampling record (16 bytes): global fall-back offset of the clamped top-left corner (channel 0 of the
// chunk is added by the reader), window-relative location + flags, and the four mask-scaled bilinear weights in bf16.
// The blend runs in packed bf16 (fma.rn.bf16x2: four roundings per sample instead of one): measured with the oracle
// on the full network this moves the end-to-end error of the bf16 engine by 1 % of itself (0.0340 -> 0.0344 relative
// rms at the 64-channel feature) and removes 60 % of the producer's instructions (no unpack, no fp32->bf16 pack).
struct __align__(16) DcnWinEntry { int goff; uint32_t meta; uint32_t w01, w23; };
constexpr uint32_t WIN_DX = 1u << 16, WIN_DY = 1u << 17, WIN_IN = 1u << 18;

// output pixel (linear b,y,x index) of GEMM row r of M tile mt; g.P_out when the row is padding
__device__ __forceinline__ int tc_pixel(const TcArgs& a, int mt, int r) {
  const ConvGeom& g = a.g;
  if (a.tiles_x == 0) { const int p = mt * TC_BM + r; return p < g.P_out ? p : g.P_out; }
  const int tpi = a.tiles_x * a.tiles_y;
  const int b = mt / tpi, t = mt - b * tpi;
  const int ty = t / a.tiles_x, tx = t - ty * a.tiles_x;
  const int oy = ty * 8 + (r >> 4), ox = tx * 16 + (r & 15);
  return (oy < g.OH && ox < g.OW) ? (b * g.OH + oy) * g.OW + ox : g.P_out;
}

// Optional timeline of the middle CTA (ct_debug_trace): clock64() stamps -- 0 start, 1 rows set up, 2 DCN table built,
// 8+s thread 0 finished gathering slice s, 5 accumulator complete, 6 epilogue done.
__device__ unsigned long long* g_tc_trace = nullptr;
// The pointer is read ONCE per thread at kernel entry (tc_trace_ptr): a stamp that re-read the global cost the stamping
// thread a dependent load per slice even with tracing off.
__device__ __forceinline__ unsigned long long* tc_trace_ptr() {
  unsigned long long* t = g_tc_trace;
  return (t != nullptr && blockIdx.x == gridDim.x / 2 && blockIdx.y == 0) ? t : nullptr;
}
__device__ __forceinline__ void tc_stamp(unsigned long long* t, int k) {
  if (t != nullptr && k < 256) t[k] = (unsigned long long)clock64();
}

// K-major, 128B-swizzled smem operand descriptor: SBO = 1024 (8 rows x 128 B), LBO unused (1).
__device__ __forceinline__ uint64_t make_sdesc(uint32_t smem_addr) {
  return wg_desc(smem_addr, 16u, 1024u, 1u);
}

// Per (tap, output pixel) DCNv2 sampling record, built once per CTA: clamped top-left corner as a 32-bit element
// offset (image base included, channel 0), element strides to the x+1 / y+1 corners (0 when that neighbour is
// outside the image, so every load address is valid and the loads need no predicate), and the four bilinear
// weights already multiplied by the modulation mask and zeroed for corners / samples outside the image.
struct __align__(16) DcnEntry { int off, dxo, dyo, pad; float w00, w01, w10, w11; };   // 32 bytes

// Sampling footprint of output pixel p (g.P_out: a padding row) for taps [tap0, tap1), the common part of both
// sampling tables: loads the 16-byte chunks of p's offset / mask row that those taps read, then calls
// f(tap, in, c, img) per tap.  in: the sample lies inside the image and c holds its footprint; img: the first pixel
// of p's image.
template <class F>
__device__ __forceinline__ void dcn_row(const TcArgs& a, int p, int tap0, int tap1, F&& f) {
  const ConvGeom& g = a.g;
  const bool ok = p < g.P_out;
  int oy = 0, ox = 0, img = 0;
  float om[28];
#pragma unroll
  for (int j = 0; j < 28; ++j) om[j] = 0.f;
  if (ok) {
    const int HWo = g.OH * g.OW;
    const int bb = p / HWo, r = p - bb * HWo;
    oy = r / g.OW; ox = r - oy * g.OW; img = bb * g.H * g.W;
    const float4* omp = reinterpret_cast<const float4*>(a.om + (size_t)p * g.ld_om);
    // offsets: floats [2 tap0, 2 tap1), masks: [18 + tap0, 18 + tap1)
#pragma unroll
    for (int j = 0; j < 7; ++j) {
      if ((4 * j < 2 * tap1 && 4 * j + 4 > 2 * tap0) || (4 * j < 18 + tap1 && 4 * j + 4 > 18 + tap0)) {
        const float4 t4 = __ldg(omp + j);
        om[4 * j] = t4.x; om[4 * j + 1] = t4.y; om[4 * j + 2] = t4.z; om[4 * j + 3] = t4.w;
      }
    }
  }
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) {
    if (tap < tap0 || tap >= tap1) continue;
    DcnCorner c;
    const bool in = ok && dcn_corner((float)(oy - 1 + tap / 3) + om[2 * tap], (float)(ox - 1 + tap % 3) + om[2 * tap + 1],
                                     g.H, g.W, om[18 + tap], c);
    f(tap, in, c, img);
  }
}

__device__ __forceinline__ uint32_t bmul2(uint32_t a, uint32_t b) {
  uint32_t d;
  asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
  return d;
}
__device__ __forceinline__ uint32_t bfma2(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t d;
  asm("fma.rn.bf16x2 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}
__device__ __forceinline__ uint32_t dup_bf2(float w) {      // {bf16(w), bf16(w)}
  uint32_t d;
  asm("cvt.rn.bf16x2.f32 %0, %1, %1;" : "=r"(d) : "f"(w));
  return d;
}

// ---- bf16x3 ("X3") engine: fp32 activations, every operand split into bf16 hi + bf16 lo = x - hi (both exact in
// fp32), and D += A_hi B_hi + A_hi B_lo + A_lo B_hi on the tensor cores with fp32 accumulation: the dropped
// A_lo B_lo term and the rounding of lo are ~2^-16 / 2^-17 relative, i.e. ~1e-5 per layer instead of bf16's 4e-3.
__device__ __forceinline__ void split8(const float4 lo4, const float4 hi4, uint4& h, uint4& l) {
  const float f[8] = {lo4.x, lo4.y, lo4.z, lo4.w, hi4.x, hi4.y, hi4.z, hi4.w};
  uint32_t hh[4], ll[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const __nv_bfloat162 hp = __floats2bfloat162_rn(f[2 * q], f[2 * q + 1]);
    const float2 hf = __bfloat1622float2(hp);
    const __nv_bfloat162 lp = __floats2bfloat162_rn(f[2 * q] - hf.x, f[2 * q + 1] - hf.y);
    hh[q] = *reinterpret_cast<const uint32_t*>(&hp);
    ll[q] = *reinterpret_cast<const uint32_t*>(&lp);
  }
  h = make_uint4(hh[0], hh[1], hh[2], hh[3]);
  l = make_uint4(ll[0], ll[1], ll[2], ll[3]);
}

// Packed bf16 blend of four corner columns with {w,w} weight pairs: mul for corner 00, then fma for 01, 10, 11.
__device__ __forceinline__ uint4 blend_bf2(const uint4 (&v)[4], uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {
  uint4 o;
  o.x = bmul2(v[0].x, w0); o.y = bmul2(v[0].y, w0); o.z = bmul2(v[0].z, w0); o.w = bmul2(v[0].w, w0);
  o.x = bfma2(v[1].x, w1, o.x); o.y = bfma2(v[1].y, w1, o.y); o.z = bfma2(v[1].z, w1, o.z); o.w = bfma2(v[1].w, w1, o.w);
  o.x = bfma2(v[2].x, w2, o.x); o.y = bfma2(v[2].y, w2, o.y); o.z = bfma2(v[2].z, w2, o.z); o.w = bfma2(v[2].w, w2, o.w);
  o.x = bfma2(v[3].x, w3, o.x); o.y = bfma2(v[3].y, w3, o.y); o.z = bfma2(v[3].z, w3, o.z); o.w = bfma2(v[3].w, w3, o.w);
  return o;
}

// One row's 8-channel column of the A operand in each activation format: its registers V, a load from global memory,
// zero, the store into a swizzled A stage of STAGE_BYTES (zeros where !live: K padding), and the DCNv2 blend of the
// four corner columns with the float weights of a DcnEntry.
struct OpBf16 {
  using T = __nv_bfloat16;
  using V = uint4;
  static constexpr uint32_t STAGE_BYTES = A_STAGE_BYTES;
  static __device__ __forceinline__ V load(const T* p) { return ldg_nc16(p); }
  static __device__ __forceinline__ V zero() { return make_uint4(0, 0, 0, 0); }
  static __device__ __forceinline__ void store(uint32_t dst, const V& v, bool live = true) {
    sts16(dst, live ? v : zero());
  }
  // same rounding points as the window sampler: weights to bf16, then the packed chain
  static __device__ __forceinline__ V blend(const V (&v)[4], const float4 w) {
    return blend_bf2(v, dup_bf2(w.x), dup_bf2(w.y), dup_bf2(w.z), dup_bf2(w.w));
  }
};
// X3: fp32 activations (channels 0-3 and 4-7), stored split into the bf16 hi tile and the lo tile A_STAGE_BYTES after
struct OpX3 {
  using T = float;
  struct V { float4 f[2]; };
  static constexpr uint32_t STAGE_BYTES = 2u * A_STAGE_BYTES;
  static __device__ __forceinline__ V load(const T* p) { return {{ldg_nc_f4(p), ldg_nc_f4(p + 4)}}; }
  static __device__ __forceinline__ V zero() { return {{make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)}}; }
  static __device__ __forceinline__ void store(uint32_t dst, const V& v, bool live = true) {
    uint4 hi, lo;
    split8(v.f[0], v.f[1], hi, lo);
    if (!live) { hi = make_uint4(0, 0, 0, 0); lo = hi; }
    sts16(dst, hi);
    sts16(dst + A_STAGE_BYTES, lo);
  }
  // fp32: w0 * v0, then fmaf for corners 1 to 3
  static __device__ __forceinline__ V blend(const V (&v)[4], const float4 w) {
    const float ww[4] = {w.x, w.y, w.z, w.w};
    V o;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      o.f[h] = make_float4(ww[0] * v[0].f[h].x, ww[0] * v[0].f[h].y, ww[0] * v[0].f[h].z, ww[0] * v[0].f[h].w);
#pragma unroll
      for (int cn = 1; cn < 4; ++cn) {
        o.f[h].x = fmaf(ww[cn], v[cn].f[h].x, o.f[h].x); o.f[h].y = fmaf(ww[cn], v[cn].f[h].y, o.f[h].y);
        o.f[h].z = fmaf(ww[cn], v[cn].f[h].z, o.f[h].z); o.f[h].w = fmaf(ww[cn], v[cn].f[h].w, o.f[h].w);
      }
    }
    return o;
  }
};

// The gather role of one thread: the 8-channel column q of GEMM rows rb + 16 i (i < TC_NROW) of every K slice, stored
// at swizzle swz into the A stages at sA.  The producers below reach the kernel's per-slice protocol through
// begin_stage(s) -> stage and end_stage(s, stage).
struct Gather { uint32_t sA, swz; int tid, q, rb, cin8, ntaps; };

// Plain convolution gather, register-prefetched two K slices ahead (8 independent 16-byte loads in flight per
// thread) while the MMAs of the previous slice run.  (tap, channel group) advance incrementally with the load order.
// row_off / row_iy / row_ix: element offset and coordinates of each row's top-left input pixel.
template <class Op, class Begin, class End>
__device__ __forceinline__ void gather_conv(const TcArgs& a, const Gather& t, const int (&row_off)[TC_NROW],
                                            const int (&row_iy)[TC_NROW], const int (&row_ix)[TC_NROW],
                                            Begin&& begin_stage, End&& end_stage) {
  using T = typename Op::T;
  using V = typename Op::V;
  const ConvGeom& g = a.g;
  int ltap = t.q / t.cin8, lcq = t.q - ltap * t.cin8;
  auto load_slice = [&](bool in_range, V (&v)[TC_NROW]) {
#pragma unroll
    for (int i = 0; i < TC_NROW; ++i) v[i] = Op::zero();
    if (in_range && ltap < t.ntaps) {
      const int ky = ltap / g.KW, kx = ltap - ky * g.KW;
      const int tap_off = (ky * g.W + kx) * g.ld_in + (lcq << 3);      // same for every row of the slice
#pragma unroll
      for (int i = 0; i < TC_NROW; ++i)
        if ((unsigned)(row_iy[i] + ky) < (unsigned)g.H && (unsigned)(row_ix[i] + kx) < (unsigned)g.W)
          v[i] = Op::load(reinterpret_cast<const T*>(a.x) + (row_off[i] + tap_off));
    }
    lcq += 8;
    while (lcq >= t.cin8) { lcq -= t.cin8; ++ltap; }
  };
  auto store_slice = [&](int s, const V (&v)[TC_NROW]) {
    const int stage = begin_stage(s);
    const uint32_t dst = t.sA + stage * Op::STAGE_BYTES + (uint32_t)t.rb * 128u + t.swz;
#pragma unroll
    for (int i = 0; i < TC_NROW; ++i) Op::store(dst + i * 2048u, v[i]);
    end_stage(s, stage);
  };
  const int KS = a.k_slices;
  V v0[TC_NROW], v1[TC_NROW];
  load_slice(0 < KS, v0);
  load_slice(1 < KS, v1);
  for (int s = 0; s < KS; s += 2) {
    store_slice(s, v0);
    load_slice(s + 2 < KS, v0);
    if (s + 1 < KS) { store_slice(s + 1, v1); load_slice(s + 3 < KS, v1); }
  }
}

// DCNv2 sampled from global memory through the DcnEntry table (CT_A_DCN).  Software-pipelined by half slices (2 of
// the thread's 4 rows): the 8 corner loads of the next half are in flight while the current half is blended.  A slice
// whose tap index runs past the kernel (K padding) samples tap 0 with its result zeroed.
template <class Op, class Begin, class End>
__device__ __forceinline__ void gather_dcn(const TcArgs& a, const Gather& t, const DcnEntry* dcn_tab,
                                           Begin&& begin_stage, End&& end_stage) {
  using T = typename Op::T;
  using V = typename Op::V;
  V va[2][4], vb[2][4];
  auto load_half = [&](int tap, int c, int half, V (&v)[2][4]) {
    const DcnEntry* tab = dcn_tab + (tap < t.ntaps ? tap : 0) * TC_BM + t.rb + 32 * half;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int4 o = *reinterpret_cast<const int4*>(&tab[16 * j]);     // off, dxo, dyo
      const T* p00 = reinterpret_cast<const T*>(a.x) + (o.x + c);
      v[j][0] = Op::load(p00);
      v[j][1] = Op::load(p00 + o.y);
      v[j][2] = Op::load(p00 + o.z);
      v[j][3] = Op::load(p00 + o.z + o.y);
    }
  };
  auto blend_half = [&](int tap, int stage, int half, const V (&v)[2][4]) {
    const bool live = tap < t.ntaps;
    const DcnEntry* tab = dcn_tab + (live ? tap : 0) * TC_BM + t.rb + 32 * half;
    const uint32_t dst = t.sA + stage * Op::STAGE_BYTES + (uint32_t)(t.rb + 32 * half) * 128u + t.swz;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const float4 w = *reinterpret_cast<const float4*>(&tab[16 * j].w00);
      Op::store(dst + j * 2048u, Op::blend(v[j], w), live);
    }
  };
  // (tap, channel group) of this thread's 8-channel column in slice s, advanced incrementally (no division)
  int tap = t.q / t.cin8, cq = t.q - tap * t.cin8;
  load_half(tap, cq << 3, 0, va);
  for (int s = 0; s < a.k_slices; ++s) {
    load_half(tap, cq << 3, 1, vb);
    const int stage = begin_stage(s);
    blend_half(tap, stage, 0, va);
    int ntap = tap, ncq = cq + 8;
    while (ncq >= t.cin8) { ncq -= t.cin8; ++ntap; }
    if (s + 1 < a.k_slices) load_half(ntap, ncq << 3, 0, va);
    blend_half(tap, stage, 1, vb);
    tap = ntap; cq = ncq;
    end_stage(s, stage);
  }
}

// DCN sampled from a shared-memory window (CT_A_DCN_WIN, bf16 only).  K order = (64-channel chunk, tap, channel): one
// K slice is one tap of one chunk, so the window of a chunk serves nine slices.  Per slice a thread blends its four
// rows' 8-channel column: 16 LDS.128 (four corners x four rows) instead of 16 L1/L2 round trips; records whose 2x2
// footprint leaves the window (offset beyond the margin) take the global path.  load_window(ch): thread 0 requests
// chunk ch of the window at s_win, completing win_bar.
template <class LoadWindow, class Begin, class End>
__device__ __forceinline__ void gather_window(const TcArgs& a, const Gather& t, const DcnWinEntry* win_tab,
                                              uint32_t s_win, uint32_t win_bar, LoadWindow&& load_window,
                                              Begin&& begin_stage, End&& end_stage) {
  const ConvGeom& g = a.g;
  const int nchunks = g.C_in >> 6;
  const uint32_t pitch = (uint32_t)a.win_pw * 128u;
  const int gdx = g.ld_in, gdy = g.W * g.ld_in;
  int s = 0;
  for (int ch = 0; ch < nchunks; ++ch) {
    mbar_wait(win_bar, (uint32_t)ch & 1u);
    for (int tap = 0; tap < 9; ++tap, ++s) {
      const int stage = begin_stage(s);
      const DcnWinEntry* tab = win_tab + tap * TC_BM + t.rb;
      uint4 e4[TC_NROW], v[TC_NROW][4];
#pragma unroll
      for (int i = 0; i < TC_NROW; ++i) e4[i] = *reinterpret_cast<const uint4*>(&tab[16 * i]);
#pragma unroll
      for (int i = 0; i < TC_NROW; ++i) {
        const uint32_t meta = e4[i].y;
        if (meta & WIN_IN) {
          const uint32_t base = s_win + ((meta & 0xffffu) << 4) + (uint32_t)(t.q << 4);
          const uint32_t dx = (meta & WIN_DX) ? 128u : 0u, dy = (meta & WIN_DY) ? pitch : 0u;
          v[i][0] = lds16(base); v[i][1] = lds16(base + dx);
          v[i][2] = lds16(base + dy); v[i][3] = lds16(base + dy + dx);
        } else {
          const __nv_bfloat16* p00 = a.x + ((int)e4[i].x + (ch << 6) + (t.q << 3));
          const int dx = (meta & WIN_DX) ? gdx : 0, dy = (meta & WIN_DY) ? gdy : 0;
          v[i][0] = ldg_nc16(p00); v[i][1] = ldg_nc16(p00 + dx);
          v[i][2] = ldg_nc16(p00 + dy); v[i][3] = ldg_nc16(p00 + dy + dx);
        }
      }
      const uint32_t dst = t.sA + stage * A_STAGE_BYTES + (uint32_t)t.rb * 128u + t.swz;
#pragma unroll
      for (int i = 0; i < TC_NROW; ++i) {
        const uint32_t w0 = __byte_perm(e4[i].z, 0, 0x1010), w1 = __byte_perm(e4[i].z, 0, 0x3232);   // {w,w} pairs
        const uint32_t w2 = __byte_perm(e4[i].w, 0, 0x1010), w3 = __byte_perm(e4[i].w, 0, 0x3232);
        sts16(dst + i * 2048u, blend_bf2(v[i], w0, w1, w2, w3));
      }
      end_stage(s, stage);
    }
    if (ch + 1 < nchunks) {                       // every thread is done with this chunk's window: refill it
      named_sync(1, TC_PRODUCERS);
      if (t.tid == 0) load_window(ch + 1);
    }
  }
}

// Output columns o0 .. o0 + 15 of pixel p (accumulator values v): + folded-BN shift, then residual / ReLU and the store
// of the output mode.  X3: fp32 NHWC activations.
template <bool X3>
__device__ __forceinline__ void tc_store16(const TcArgs& a, int p, int o0, float (&v)[16]) {
  const ConvGeom& g = a.g;
  if (a.shift) {
    if (o0 + 16 <= g.C_out && (reinterpret_cast<size_t>(a.shift + o0) & 15) == 0) {   // four 16-byte loads
      const float4* sh4 = reinterpret_cast<const float4*>(a.shift + o0);
#pragma unroll
      for (int j4 = 0; j4 < 4; ++j4) {
        const float4 sh = __ldg(sh4 + j4);
        v[4 * j4] += sh.x; v[4 * j4 + 1] += sh.y; v[4 * j4 + 2] += sh.z; v[4 * j4 + 3] += sh.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j) if (o0 + j < g.C_out) v[j] += __ldg(a.shift + o0 + j);
    }
  }
  if (X3 && g.out_mode == CT_OUT_NHWC) {            // fp32 activations in, fp32 activations out
    const float* res = a.residual ? reinterpret_cast<const float*>(a.residual) + (size_t)p * g.ld_res + o0 : nullptr;
    store_f32_act16(reinterpret_cast<float*>(a.out) + (size_t)p * g.ld_out + o0, v, res, g.relu);
  } else if (g.out_mode == CT_OUT_NHWC) {
    if (a.residual) {
      const uint4* rp = reinterpret_cast<const uint4*>(a.residual + (size_t)p * g.ld_res + o0);
      const uint4 ra = ldg_nc16(rp), rb2 = ldg_nc16(rp + 1);
      add_residual_bf16(v, ra, rb2);
    }
    relu16(v, g.relu);
    store_bf16x16(reinterpret_cast<__nv_bfloat16*>(a.out) + (size_t)p * g.ld_out + o0, v);
  } else if (g.out_mode == CT_OUT_NHWC_F32) {
    store_f32_nhwc16(reinterpret_cast<float*>(a.out) + (size_t)p * g.ld_out + o0, v, o0, g);
  } else {
    const int HWo = g.OH * g.OW;
    const int b = p / HWo, rr = p - b * HWo;
    store_head16(reinterpret_cast<float*>(a.out) + ((size_t)b * g.C_out + o0) * HWo + rr, HWo, v, o0, g);
  }
}

template <bool X3, int N>
__global__ void __launch_bounds__(TC_THREADS, (!X3 && N <= 64) ? 2 : 1)
conv_tc_kernel(const TcArgs a, const __grid_constant__ CUtensorMap tmap) {
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  // SWIZZLE_128B operands need 1024B-aligned stage bases: align by hand (launch adds 1 KB of slack)
  unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  const ConvGeom& g = a.g;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = tid >> 7;                 // warpgroup: GEMM rows 64 wg .. 64 wg + 63
  unsigned long long* const trace = tc_trace_ptr();
  const int S = a.stages;
  constexpr uint32_t b_tile_bytes = (uint32_t)N * 128u;                       // one bf16 weight tile of a K slice
  constexpr uint32_t b_stage_bytes = X3 ? 2u * b_tile_bytes : b_tile_bytes;   // X3: [hi][lo]
  using Op = std::conditional_t<X3, OpX3, OpBf16>;
  constexpr uint32_t a_stage_bytes = Op::STAGE_BYTES;                         // X3: [hi 16 KB][lo 16 KB]

  // carve shared memory: [stages | epilogue staging][barriers][DCN table / window]
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t sA = smem_base;
  const uint32_t sB = sA + S * a_stage_bytes;
  const uint32_t off_bar = a.region0;
  const uint32_t bars = smem_base + off_bar;           // full[S], empty[S], win_full
  DcnEntry* dcn_tab = reinterpret_cast<DcnEntry*>(smem + off_bar + (2 * S + 1) * 8 + 24);  // 16B aligned
  auto full_bar = [&](int s) { return bars + 8u * s; };
  auto empty_bar = [&](int s) { return bars + 8u * (S + s); };
  const uint32_t win_bar = bars + 8u * (2 * S);
  const bool win = !X3 && a.a_mode == CT_A_DCN_WIN;
  // CT_A_DCN_WIN: [table 9 x 128 x 16 B][window, 128B aligned]
  DcnWinEntry* win_tab = reinterpret_cast<DcnWinEntry*>(dcn_tab);
  const uint32_t s_win = (smem_u32(dcn_tab) + 9u * TC_BM * 16u + 127u) & ~127u;

  const int mt = blockIdx.x;
  const int nt = blockIdx.y;
  const int n0 = nt * N;
  if (tid == 0) tc_stamp(trace, 0);
  pdl_trigger();                       // the next kernel of the stream may start its own prologue now

  if (tid == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), TC_THREADS / 32); }
    mbar_init(win_bar, 1);
    mbar_init_fence();
  }
  __syncthreads();
  pdl_wait();                          // everything below reads what the previous kernel wrote

  // =========================== A gather (both warpgroups) ===========================
  const int q = tid & 7;                   // 16-byte chunk (8 channels) inside the 64-wide K slice
  const int rb = wg * 64 + ((tid & 127) >> 3);   // rows rb + 16*i, i < TC_NROW
  const uint32_t swz = (uint32_t)((q ^ (rb & 7)) << 4);
  const int HWo = g.OH * g.OW;
  int row_off[TC_NROW], row_iy[TC_NROW], row_ix[TC_NROW];   // element offset / coords of the window's top-left input pixel
  if (a.a_mode != CT_A_CONV) {
    // DCN rows come from the sampling table
#pragma unroll
    for (int i = 0; i < TC_NROW; ++i) { row_off[i] = 0; row_iy[i] = -100000; row_ix[i] = -100000; }
  } else if (a.tiles_x != 0) {
#pragma unroll
    for (int i = 0; i < TC_NROW; ++i) {
      const int p = tc_pixel(a, mt, rb + 16 * i);
      if (p < g.P_out) {
        const int b = p / HWo, r = p - b * HWo;
        const int oy = r / g.OW, ox = r - oy * g.OW;
        row_iy[i] = oy * g.stride - g.pad;
        row_ix[i] = ox * g.stride - g.pad_w;
        row_off[i] = (b * g.H * g.W + row_iy[i] * g.W + row_ix[i]) * g.ld_in;
      } else {
        row_off[i] = 0; row_iy[i] = -100000; row_ix[i] = -100000;
      }
    }
  } else {
    // linear tiles: one division pair for the first row, the other rows (+16 pixels each) by carry propagation
    int p = mt * TC_BM + rb;
    int b = p / HWo, r = p - b * HWo;
    int oy = r / g.OW, ox = r - oy * g.OW;
#pragma unroll
    for (int i = 0; i < TC_NROW; ++i) {
      if (p < g.P_out) {
        row_iy[i] = oy * g.stride - g.pad;
        row_ix[i] = ox * g.stride - g.pad_w;
        row_off[i] = (b * g.H * g.W + row_iy[i] * g.W + row_ix[i]) * g.ld_in;
      } else {
        row_off[i] = 0; row_iy[i] = -100000; row_ix[i] = -100000;
      }
      p += 16; ox += 16;
      while (ox >= g.OW) { ox -= g.OW; ++oy; }
      while (oy >= g.OH) { oy -= g.OH; ++b; }
    }
  }
  if (tid == 0) tc_stamp(trace, 1);
  int win_x0 = 0, win_y0 = 0, win_b = 0;
  auto load_window = [&](int ch) {                    // 64-channel chunk ch of the window: TMA, zero fill outside
    mbar_arrive_expect_tx(win_bar, a.win_bytes);      // count 1: this arrival + the TMA's bytes complete the phase
    tma_4d(s_win, &tmap, ch << 6, win_x0, win_y0, win_b, win_bar);
  };
  if (win) {
    // window origin of this 8x16 patch: one kernel-halo pixel + the offset margin to the top/left
    const int tpi = a.tiles_x * a.tiles_y;
    win_b = mt / tpi;
    const int t = mt - win_b * tpi;
    const int ty = t / a.tiles_x, tx = t - ty * a.tiles_x;
    win_y0 = ty * 8 - 1 - a.win_m;
    win_x0 = tx * 16 - 1 - a.win_m;
    if (tid == 0) load_window(0);
    // Two threads per row (taps 0-4 and 5-8).  The 27 offset / mask floats of a row sit in one 128-byte line of `om`;
    // each thread loads only the 16-byte chunks its taps need.
    const int trow = tid & (TC_BM - 1), thalf = tid >> 7;            // thalf 0: taps 0..4, thalf 1: taps 5..8
    dcn_row(a, tc_pixel(a, mt, trow), thalf ? 5 : 0, thalf ? 9 : 5, [&](int tap, bool in, const DcnCorner& c, int img) {
      DcnWinEntry e; e.goff = 0; e.meta = WIN_IN; e.w01 = 0u; e.w23 = 0u;
      if (in) {
        e.goff = (img + c.yc * g.W + c.xc) * g.ld_in;
        const bool inside = c.y0 >= win_y0 && c.y0 + 1 <= win_y0 + a.win_ph - 1 && c.x0 >= win_x0 &&
                            c.x0 + 1 <= win_x0 + a.win_pw - 1;
        const uint32_t woff16 = (uint32_t)((c.yc - win_y0) * a.win_pw + (c.xc - win_x0)) * 8u;   // 128 B per pixel
        e.meta = (inside ? (woff16 | WIN_IN) : 0u) | (c.dx ? WIN_DX : 0u) | (c.dy ? WIN_DY : 0u);
        const __nv_bfloat162 wa = __floats2bfloat162_rn(c.w00, c.w01), wb = __floats2bfloat162_rn(c.w10, c.w11);
        e.w01 = *reinterpret_cast<const uint32_t*>(&wa);
        e.w23 = *reinterpret_cast<const uint32_t*>(&wb);
      }
      win_tab[tap * TC_BM + trow] = e;
    });
    named_sync(1, TC_PRODUCERS);
    if (tid == 0) tc_stamp(trace, 2);
  }
  if (a.a_mode == CT_A_DCN) {
    // per (tap,row) sampling records, computed once per CTA (row = tid, threads 0..127)
    if (tid < TC_BM) {
      dcn_row(a, tc_pixel(a, mt, tid), 0, 9, [&](int tap, bool in, const DcnCorner& c, int img) {
        DcnEntry e; e.off = 0; e.dxo = 0; e.dyo = 0; e.pad = 0; e.w00 = e.w01 = e.w10 = e.w11 = 0.f;
        if (in) {
          e.off = (img + c.yc * g.W + c.xc) * g.ld_in;
          e.dxo = c.dx ? g.ld_in : 0;
          e.dyo = c.dy ? g.W * g.ld_in : 0;
          e.w00 = c.w00; e.w01 = c.w01; e.w10 = c.w10; e.w11 = c.w11;
        }
        dcn_tab[tap * TC_BM + tid] = e;
      });
    }
    named_sync(1, TC_PRODUCERS);
    if (tid == 0) tc_stamp(trace, 2);
  }
  const size_t w_slice_elems = (size_t)(X3 ? 2 : 1) * N * TC_BK;
  const __nv_bfloat16* wt = a.w + (size_t)nt * a.k_slices * w_slice_elems;

  // ---- per-slice protocol.  begin: wait until both warpgroups' MMAs of the slice that last used the stage are done
  // (empty barrier, one arrival per warp), then thread 0 requests the weight tile.  end: the warpgroup's A rows are
  // made visible to the async proxy, the warpgroup synchronises, waits for the weight tile and issues its MMAs; after
  // those of the PREVIOUS slice have completed (wait_group 1) each warp releases that slice's stage.
  float acc[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
  auto begin_stage = [&](int s) {
    const int stage = s % S;
    const uint32_t ph = (uint32_t)(s / S) & 1u;
    mbar_wait(empty_bar(stage), ph ^ 1u);
    if (tid == 0) {
      mbar_arrive_expect_tx(full_bar(stage), b_stage_bytes);
      bulk_g2s(sB + stage * b_stage_bytes, wt + (size_t)s * w_slice_elems, b_stage_bytes, full_bar(stage));
    }
    return stage;
  };
  auto end_stage = [&](int s, int stage) {
    fence_proxy_async();                 // generic-proxy smem writes -> visible to the tensor-core (async) proxy
    named_sync(2 + wg, 128);
    mbar_wait(full_bar(stage), (uint32_t)(s / S) & 1u);
    if (tid == 0) tc_stamp(trace, 8 + s);
    const uint32_t a_base = sA + stage * a_stage_bytes + (uint32_t)wg * (64u * 128u);
    const uint64_t ad = make_sdesc(a_base);
    const uint64_t bd = make_sdesc(sB + stage * b_stage_bytes);
    wg_fence();
    if constexpr (X3) {
      const uint64_t ad_lo = make_sdesc(a_base + A_STAGE_BYTES);
      const uint64_t bd_lo = make_sdesc(sB + stage * b_stage_bytes + b_tile_bytes);
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k) {      // small cross terms first, then the hi x hi term
        Wgmma<N>::mma(acc, ad_lo + 2ull * k, bd + 2ull * k, (s > 0 || k > 0) ? 1u : 0u);
        Wgmma<N>::mma(acc, ad + 2ull * k, bd_lo + 2ull * k, 1u);
        Wgmma<N>::mma(acc, ad + 2ull * k, bd + 2ull * k, 1u);
      }
    } else {
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k)
        Wgmma<N>::mma(acc, ad + 2ull * k, bd + 2ull * k, (s > 0 || k > 0) ? 1u : 0u);
    }
    wg_commit();
    wg_wait<1>();
    wg_fence_operand(acc);
    if (s > 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar((s - 1) % S));
    }
  };

  const Gather t{sA, swz, tid, q, rb, g.C_in >> 3, g.KH * g.KW};
  if (win) gather_window(a, t, win_tab, s_win, win_bar, load_window, begin_stage, end_stage);
  else if (a.a_mode == CT_A_DCN) gather_dcn<Op>(a, t, dcn_tab, begin_stage, end_stage);
  else gather_conv<Op>(a, t, row_off, row_iy, row_ix, begin_stage, end_stage);
  wg_wait<0>();
  wg_fence_operand(acc);
  if (tid == 0) tc_stamp(trace, 5);
  __syncthreads();                     // every MMA has read its stage: the stage area becomes the staging tile

  // =========================== epilogue ===========================
  // 32 accumulator columns at a time through shared memory; thread (warp w, lane l) then owns GEMM row 32 (w % 4) + l
  // and the 16-column half w / 4 of the chunk.
  const uint32_t stg = sA;
  const int wq = warp & 3, chalf = warp >> 2;
  const int row = wq * 32 + lane;
  const int p = tc_pixel(a, mt, row);
  const bool p_ok = p < g.P_out;
#pragma unroll
  for (int c0 = 0; c0 < N; c0 += 32) {
    stage_acc_chunk(acc, c0, stg, wg * 64);
    __syncthreads();
    const int col = c0 + chalf * 16;
    const int o0 = n0 + col;
    if (col < N && p_ok && o0 < g.C_out) {
      float v[16];
      lds_f(stg + ((uint32_t)row * EPI_PITCH + (uint32_t)chalf * 16u) * 4u, v);
      tc_store16<X3>(a, p, o0, v);
    }
    __syncthreads();
  }
  if (tid == 0) tc_stamp(trace, 6);
}

// ---- plain convolutions of the bf16 engine with C_in % 64 == 0: TMA-fed, persistent, warp-specialised ----
// K order as above (k = tap * C_in + c): K slice s is one tap of one 64-channel chunk, so the A operand of a slice is ONE
// tensor-map box {64 channels, 16 x, 8 y, 1 image} at (c0, ox0 * stride - pad_w + kx, oy0 * stride - pad + ky, b): its 128
// rows of 128 bytes land in tc_pixel's 8 x 16 patch order, 128B-swizzled, i.e. exactly the K-major layout make_sdesc
// describes.  The map's zero fill is the padding, its element strides (= stride in x and y) the strided convolutions,
// and its channel stride ld_in reads channel slices of wider (concat) buffers in place.
//
// Two warpgroups issue the MMAs of GEMM rows 64 w .. 64 w + 63 and then store them (tc_store16); one arrival per warp on
// the empty barrier releases a stage.  Thread 0 issues the A box and the weight tile of each slice into one stage, both
// completing the stage's full barrier: S slices up front, then one per released stage, S - 1 slices ahead of the MMAs.
// CTAs are persistent (static stride over the (m, n) tiles), so these loads run into the next tile's slices while the
// warpgroups finish the current one; at N <= 128 two CTAs share an SM and one CTA's epilogue runs under the other's MMAs.
// (A separate producer warp would make 9 warps per CTA: the register file of an SM sub-partition then holds two such
// CTAs only at 96 registers, where N = 128 spills.)
// The epilogue stages 16 accumulator columns at a time (10 KB for both warpgroups instead of 18 KB for 32 columns): that
// is what lets N = 128 hold 3 stages and N <= 64 hold 4 within the 113 KB of a CTA at two CTAs per SM.
constexpr int TMA_THREADS = 256;
constexpr int TMA_EPI_COLS = 16;
constexpr int TMA_EPI_PITCH = TMA_EPI_COLS + 4;               // floats per staging row: 16-byte reads conflict-free
constexpr int TMA_STAGING_BYTES = 2 * 64 * TMA_EPI_PITCH * 4; // per warpgroup: 64 rows x 16 columns of fp32

template <int N>
__global__ void __launch_bounds__(TMA_THREADS, N <= 128 ? 2 : 1)
conv_tma_kernel(const TcArgs a, const __grid_constant__ CUtensorMap tmap) {
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  const ConvGeom& g = a.g;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int S = a.stages;
  constexpr uint32_t b_bytes = (uint32_t)N * 128u;
  // smem: [A stages][B stages][staging 2 x 64 x TMA_EPI_PITCH fp32][full[S], empty[S]]
  const uint32_t sA = smem_u32(smem);
  const uint32_t sB = sA + S * A_STAGE_BYTES;
  const uint32_t sStg = sB + S * b_bytes;
  const uint32_t bars = sStg + TMA_STAGING_BYTES;
  auto full_bar = [&](int s) { return bars + 8u * s; };
  auto empty_bar = [&](int s) { return bars + 8u * (S + s); };
  const int m_tiles = g.B * a.tiles_x * a.tiles_y;
  const int items = m_tiles * ((g.C_out + N - 1) / N);
  const int KS = a.k_slices;

  pdl_trigger();
  if (tid == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 8); }
    mbar_init_fence();
  }
  __syncthreads();
  pdl_wait();

  // ---- loads (thread 0): the next slice (l_item, l_s) of this CTA's items, into stage l_it % S once it is empty
  int l_item = blockIdx.x, l_s = 0, l_it = 0;
  auto load_next = [&]() {
    if (l_item >= items) return;
    const int stage = l_it % S;
    mbar_wait(empty_bar(stage), ((uint32_t)(l_it / S) & 1u) ^ 1u, 1, l_it);
    const int nt = l_item / m_tiles, mt = l_item - nt * m_tiles;
    const int tpi = a.tiles_x * a.tiles_y;
    const int b = mt / tpi, t = mt - b * tpi;
    const int ty = t / a.tiles_x, tx = t - ty * a.tiles_x;
    const int nch = g.C_in >> 6;
    const int tap = l_s / nch, ch = l_s - tap * nch;
    const int ky = tap / g.KW, kx = tap - ky * g.KW;
    mbar_arrive_expect_tx(full_bar(stage), (uint32_t)A_STAGE_BYTES + b_bytes);
    tma_4d(sA + stage * A_STAGE_BYTES, &tmap, ch << 6, tx * 16 * g.stride - g.pad_w + kx,
           ty * 8 * g.stride - g.pad + ky, b, full_bar(stage));
    bulk_g2s(sB + stage * b_bytes, a.w + ((size_t)nt * KS + l_s) * (N * TC_BK), b_bytes, full_bar(stage));
    ++l_it;
    if (++l_s == KS) { l_s = 0; l_item += gridDim.x; }
  };
  if (tid == 0)
    for (int i = 0; i < S; ++i) load_next();

  // ===================== MMA + epilogue warpgroups =====================
  const int wg = warp >> 2, w4 = warp & 3;
  const int lrow = 32 * (w4 & 1) + lane;           // epilogue: row of this warpgroup's 64, 16-column half chalf
  const int chalf = w4 >> 1;
  const uint32_t stg = sStg + (uint32_t)wg * (64u * TMA_EPI_PITCH * 4u);
  float acc[N / 2];
  int it = 0;
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int nt = item / m_tiles, mt = item - nt * m_tiles;
    for (int s = 0; s < KS; ++s, ++it) {
      const int stage = it % S;
      mbar_wait(full_bar(stage), (uint32_t)(it / S) & 1u, 2, it);
      const uint64_t ad = make_sdesc(sA + stage * A_STAGE_BYTES + (uint32_t)wg * (64u * 128u));
      const uint64_t bd = make_sdesc(sB + stage * b_bytes);
      wg_fence();
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k)
        Wgmma<N>::mma(acc, ad + 2ull * k, bd + 2ull * k, (s > 0 || k > 0) ? 1u : 0u);
      wg_commit();
      wg_wait<1>();
      wg_fence_operand(acc);
      if (s > 0) {                                   // the previous slice's MMAs are done with its stage
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar((it - 1) % S));
        if (tid == 0) load_next();
      }
    }
    wg_wait<0>();
    wg_fence_operand(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(empty_bar((it - 1) % S));
    if (tid == 0) load_next();

    // ---- epilogue of this warpgroup's 64 rows, 32 accumulator columns at a time: the two 16-column halves pass in turn
    // through the staging tile, half h read by the threads with chalf == h, then every thread stores its 16 columns
    const int p = tc_pixel(a, mt, 64 * wg + lrow);
    const bool p_ok = p < g.P_out;
    const int n0 = nt * N;
#pragma unroll
    for (int c0 = 0; c0 < N; c0 += 32) {
      float v[16];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        named_sync(1 + wg, 128);                   // the previous half's readers are done with the staging tile
        stage_acc_chunk<N / 2, TMA_EPI_COLS, TMA_EPI_PITCH>(acc, c0 + h * TMA_EPI_COLS, stg, 0);
        named_sync(1 + wg, 128);
        if (chalf == h) lds_f(stg + (uint32_t)lrow * TMA_EPI_PITCH * 4u, v);
      }
      const int col = c0 + chalf * 16;
      const int o0 = n0 + col;
      if (col < N && p_ok && o0 < g.C_out) tc_store16<false>(a, p, o0, v);
    }
  }
}

int tc_set_trace(void* buf) {
  unsigned long long* p = (unsigned long long*)buf;
  return cudaMemcpyToSymbol(g_tc_trace, &p, sizeof(p)) == cudaSuccess ? CT_OK : CT_ERR_CUDA;
}
int tc_set_watch(void* mapped_host_buf) { return set_mbar_watch(mapped_host_buf); }

// Plain bf16 convolutions whose K slices are whole 64-channel chunks of one tap take conv_tma_kernel when its 8 x 16
// patches cover the output map with at most 15 % of padding rows; the others (C_in not a multiple of 64, maps such as
// mot's 34 x 60 / 17 x 30, the bf16x3 engine) the register gather of conv_tc_kernel, whose 128-pixel tiles run across
// image rows and images.
static bool tc_uses_tma(const ct_conv_desc* d) {
  if (d->engine != CT_ENGINE_TCGEN05 || d->a_mode != CT_A_CONV || d->C_in % 64 != 0 || d->stride < 1 || d->stride > 8)
    return false;
  const long long padded = (long long)((d->OW + 15) / 16) * ((d->OH + 7) / 8) * 128;
  return (long long)d->OH * d->OW * 100 >= padded * 85;
}

// Configuration step: the launch arguments other than the pointers, and the launch configuration.  No CUDA call.
static int tc_config(const ct_conv_desc* d, TcArgs& a, ConvConfig& c) {
  const bool x3 = d->engine == CT_ENGINE_TCGEN05_X3;     // fp32 activations, bf16 hi/lo split operands
  a.g = make_geom(d);
  const ConvGeom& g = a.g;
  if (g.C_in % 8 != 0 || g.ld_in % 8 != 0)
    return fail(CT_ERR_INVALID, "conv_tc: C_in and ld_in must be multiples of 8%s (%ld,%ld)", "", g.C_in, g.ld_in);
  const int n_tile = d->n_tile;
  if (n_tile <= 0 || n_tile % 16 != 0 || n_tile > 256)
    return fail(CT_ERR_INVALID, "conv_tc: n_tile must be a multiple of 16 in [16,256]%s (%ld)", "", n_tile);
  if (g.out_mode == CT_OUT_NHWC) {
    if (g.C_out % 16 != 0 || g.ld_out % 8 != 0)
      return fail(CT_ERR_INVALID, "conv_tc: NHWC output needs C_out %% 16 == 0 and ld_out %% 8 == 0%s", "");
    if (d->residual && g.ld_res % 8 != 0)
      return fail(CT_ERR_INVALID, "conv_tc: residual needs ld_res %% 8 == 0%s", "");
  } else if (d->residual) {
    return fail(CT_ERR_INVALID, "conv_tc: residual unsupported for fp32 outputs%s", "");
  }
  if ((long long)g.B * g.H * g.W * g.ld_in >= (1ll << 31))
    return fail(CT_ERR_INVALID, "conv_tc: input tensor exceeds 2^31 elements (32-bit offsets)%s", "");
  a.n_tile = n_tile;
  a.k_slices = (g.K_total + TC_BK - 1) / TC_BK;
  a.a_mode = d->a_mode;
  // CT_A_DCN_WIN needs 64-channel chunks and the bf16 engine; anything else samples from global memory (same results:
  // for C_in == 64 the two K orders coincide, otherwise the caller packed the weights chunk-major and must get WIN)
  const bool win = d->a_mode == CT_A_DCN_WIN;
  if (win && (x3 || g.C_in % 64 != 0))
    return fail(CT_ERR_INVALID, "conv_tc: CT_A_DCN_WIN needs the bf16 engine and C_in %% 64 == 0%s (%ld)", "", g.C_in);
  // dcn_row reads a pixel's offset / mask row as 16-byte vectors: consecutive rows must stay 16 bytes apart
  if (d->a_mode != CT_A_CONV && g.ld_om % 4 != 0)
    return fail(CT_ERR_INVALID, "conv_tc: DCN needs ld_om %% 4 == 0 (16-byte offset / mask rows)%s (%ld)", "", g.ld_om);
  static const int win_margin = getenv("CTB_TC_DCN_MARGIN") ? atoi(getenv("CTB_TC_DCN_MARGIN")) : 2;
  a.win_m = win_margin < 0 ? 0 : (win_margin > 6 ? 6 : win_margin);
  a.win_pw = 16 + 2 * a.win_m + 3;
  a.win_ph = 8 + 2 * a.win_m + 3;
  a.win_bytes = (uint32_t)(a.win_pw * a.win_ph * 128);
  if (tc_uses_tma(d)) {
    // as many stages (up to 4) as fit in the CTA's share of the SM: half of it at N <= 128 (two CTAs per SM)
    const size_t stage = (size_t)A_STAGE_BYTES + (size_t)n_tile * 128;
    const size_t limit = (n_tile <= 128 ? 113 : 227) * 1024;
    auto smem_for = [&](int stg) { return (size_t)stg * stage + TMA_STAGING_BYTES + 2 * stg * 8 + 1024; };
    int stages = 4;
    while (stages > 2 && smem_for(stages) > limit) --stages;
    if (smem_for(stages) > limit)
      return fail(CT_ERR_UNSUPPORTED, "conv_tc: tile does not fit in shared memory%s (%ld)", "", (long)smem_for(stages));
    a.stages = stages;
    a.region0 = 0;
    a.tiles_x = (g.OW + 15) / 16;
    a.tiles_y = (g.OH + 7) / 8;
    c.smem_bytes = (int32_t)smem_for(stages);
    c.stages = stages;
    c.tile_w = 16;
    c.tile_h = 8;
    c.ctas_per_sm = 0;
    c.overlap = 0;
    return CT_OK;
  }
  const size_t stage_bytes = (size_t)(x3 ? 2 : 1) * (A_STAGE_BYTES + n_tile * 128);
  const size_t staging = (size_t)TC_BM * EPI_PITCH * 4;      // <= one stage (16 KB + n_tile x 128 B)
  auto region0_for = [&](int stg) { return ((size_t)stg * stage_bytes > staging ? (size_t)stg * stage_bytes : staging); };
  auto smem_for = [&](int stg) {
    return region0_for(stg) + (2 * stg + 1) * 8 + 32 +
           (d->a_mode == CT_A_DCN ? 9 * TC_BM * sizeof(DcnEntry) : 0) +
           (win ? 9 * TC_BM * sizeof(DcnWinEntry) + 128 + a.win_bytes : 0) + 1024;
  };
  // The MMAs of a slice overlap the gather of the next one, so two stages keep the tensor cores fed; a third covers
  // the weight-tile copy.  Narrow tiles keep two CTAs per SM (<= 113 KB each).
  int stages = 3;
  if (smem_for(stages) > 113 * 1024 && smem_for(2) <= 113 * 1024) stages = 2;
  if (d->a_mode == CT_A_DCN) {
    // the DCN gather, not the MMA, paces the pipeline: fewer stages leave more of the SM's shared memory to L1, which
    // the bilinear corner reads (each input pixel is touched ~36 times) depend on
    static const int dcn_stages = getenv("CTB_TC_DCN_STAGES") ? atoi(getenv("CTB_TC_DCN_STAGES")) : 2;
    if (dcn_stages >= 2 && dcn_stages < stages) stages = dcn_stages;
  }
  if (win) {
    static const int win_stages = getenv("CTB_TC_WIN_STAGES") ? atoi(getenv("CTB_TC_WIN_STAGES")) : 0;
    stages = 2;
    if (win_stages >= 2) stages = win_stages;
  }
  while (stages > 2 && smem_for(stages) > 227 * 1024) --stages;
  if (smem_for(stages) > 227 * 1024)
    return fail(CT_ERR_UNSUPPORTED, "conv_tc: tile does not fit in shared memory%s (%ld)", "", (long)smem_for(stages));
  if (stages > a.k_slices) stages = a.k_slices;
  a.stages = stages;
  a.region0 = (uint32_t)region0_for(stages);
  // M tiles: 128 consecutive pixels, or 8 (y) x 16 (x) patches -- always for the window sampler (ragged at the right /
  // bottom edge), and with CTB_TC_TILE2D=1 (off by default) where they tile the map exactly.
  static const int tile2d_env = getenv("CTB_TC_TILE2D") ? atoi(getenv("CTB_TC_TILE2D")) : 0;
  a.tiles_x = a.tiles_y = 0;
  if (win || (tile2d_env && g.OW % 16 == 0 && g.OH % 8 == 0)) {
    a.tiles_x = (g.OW + 15) / 16;
    a.tiles_y = (g.OH + 7) / 8;
  }
  c.smem_bytes = (int32_t)smem_for(stages);
  c.stages = stages;
  c.tile_w = a.tiles_x ? 16 : TC_BM;
  c.tile_h = a.tiles_x ? 8 : 1;
  c.ctas_per_sm = 0;
  c.overlap = 0;
  return CT_OK;
}

int conv_config_tc(const ct_conv_desc* d, ConvConfig* c) {
  TcArgs a;
  return tc_config(d, a, *c);
}

int conv_forward_tc(const ct_conv_desc* d, cudaStream_t st) {
  TcArgs a;
  ConvConfig c;
  const int rc = tc_config(d, a, c);
  if (rc != CT_OK) return rc;
  if (((uintptr_t)d->x & 15) || ((uintptr_t)d->w & 15) || ((uintptr_t)d->out & 15) || ((uintptr_t)d->residual & 15))
    return fail(CT_ERR_INVALID, "conv_tc: x/w/out/residual must be 16-byte aligned%s", "");
  if (d->a_mode != CT_A_CONV && ((uintptr_t)d->om & 15))
    return fail(CT_ERR_INVALID, "conv_tc: DCN needs a 16-byte aligned om%s", "");
  a.x = (const __nv_bfloat16*)d->x;
  a.w = (const __nv_bfloat16*)d->w;
  a.shift = d->shift;
  a.residual = (const __nv_bfloat16*)d->residual;
  a.om = d->om;
  a.out = d->out;
  const ConvGeom& g = a.g;
  const int m_tiles = a.tiles_x ? g.B * a.tiles_x * a.tiles_y : (g.P_out + TC_BM - 1) / TC_BM;
  const int n_tiles = (g.C_out + a.n_tile - 1) / a.n_tile;
  CUtensorMap tmap;
  memset(&tmap, 0, sizeof(tmap));
  const cuuint64_t dims[4] = {(cuuint64_t)g.C_in, (cuuint64_t)g.W, (cuuint64_t)g.H, (cuuint64_t)g.B};
  const cuuint64_t strides[3] = {(cuuint64_t)g.ld_in * 2, (cuuint64_t)g.W * g.ld_in * 2, (cuuint64_t)g.H * g.W * g.ld_in * 2};
  if (tc_uses_tma(d)) {
    // one K slice of an 8 x 16 output patch: 64 channels of 16 x 8 input pixels `stride` apart (the box counts elements
    // before striding)
    const cuuint32_t s = (cuuint32_t)g.stride;
    const cuuint32_t box[4] = {64, 16 * s, 8 * s, 1};
    const cuuint32_t estr[4] = {1, s, s, 1};
    const int r = encode_tmap_bf16(&tmap, d->x, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B, estr);
    if (r != CT_OK) return r;
    const int items = m_tiles * n_tiles;
    const int per_sm = a.n_tile <= 128 ? 2 : 1;
    const int grid = items < device_sm_count() * per_sm ? items : device_sm_count() * per_sm;
    return dispatch_n_tile(a.n_tile, [&](auto n) {
      constexpr int N = decltype(n)::value;
      return launch_big_smem<conv_tma_kernel<N>>(dim3(grid), dim3(TMA_THREADS), c.smem_bytes, st, a, tmap);
    });
  }
  if (a.a_mode == CT_A_DCN_WIN) {                    // the TMA box of one patch's window
    const cuuint32_t box[4] = {64, (cuuint32_t)a.win_pw, (cuuint32_t)a.win_ph, 1};
    const int r = encode_tmap_bf16(&tmap, d->x, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE);
    if (r != CT_OK) return r;
  }
  dim3 grid(m_tiles, n_tiles);
  const bool x3 = d->engine == CT_ENGINE_TCGEN05_X3;
  return dispatch_n_tile(a.n_tile, [&](auto n) {
    constexpr int N = decltype(n)::value;
    return x3 ? launch_big_smem<conv_tc_kernel<true, N>>(grid, dim3(TC_THREADS), c.smem_bytes, st, a, tmap)
              : launch_big_smem<conv_tc_kernel<false, N>>(grid, dim3(TC_THREADS), c.smem_bytes, st, a, tmap);
  });
}

}  // namespace ctb
