// fp32-accumulate SIMT implicit-GEMM convolution / DCNv2 ("precise" engine).
// One kernel covers every conv-like layer of the path (see ctb200.h: ct_conv_forward).  It is the
// reference-accuracy CUDA path (fp32 activations -> matches the reference within 1e-3 end to end)
// and the on-device cross-check for the wgmma engine (same packing order k = tap*C_in + c).
//
// Tile: 64 output pixels x 64 output channels per CTA, K step 16, 256 threads, 4x4 outputs/thread.
#include "conv_common.cuh"

namespace ctb {

constexpr int BM = 64, BN = 64, BK = 16, NT = 256;

template <typename T> struct Vec4;
template <> struct Vec4<float> {
  static __device__ __forceinline__ float4 ld(const float* p) {
    return __ldg(reinterpret_cast<const float4*>(p));
  }
};
template <> struct Vec4<__nv_bfloat16> {
  static __device__ __forceinline__ float4 ld(const __nv_bfloat16* p) {
    const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
    const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(&u.x);
    const __nv_bfloat162 b = *reinterpret_cast<const __nv_bfloat162*>(&u.y);
    const float2 fa = __bfloat1622float2(a), fb = __bfloat1622float2(b);
    return make_float4(fa.x, fa.y, fb.x, fb.y);
  }
};

template <typename T, int AMODE>
__global__ void __launch_bounds__(NT)
conv_simt_kernel(ConvGeom g, const T* __restrict__ x, const float* __restrict__ w, int ldw,
                 const float* __restrict__ shift, const T* __restrict__ residual,
                 const float* __restrict__ om, void* __restrict__ out) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN];

  const int t = threadIdx.x;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;

  // A-load role: pixel (t>>2) of the tile, channel quad (t&3) of the 16-wide K step
  const int am = t >> 2, aq = t & 3;
  const int ap = m0 + am;
  const bool a_ok = ap < g.P_out;
  int ab = 0, aoy = 0, aox = 0;
  if (a_ok) {
    ab = ap / (g.OH * g.OW);
    const int r = ap - ab * g.OH * g.OW;
    aoy = r / g.OW; aox = r - aoy * g.OW;
  }
  const T* xb = x + (size_t)ab * g.H * g.W * g.ld_in;
  const float* om_px = (AMODE == CT_A_DCN && a_ok) ? om + (size_t)ap * g.ld_om : nullptr;

  // B-load role
  const int bk = t >> 4, bo = (t & 15) * 4;

  const int tm = t >> 4, tn = t & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < g.K_total; k0 += BK) {
    // ---- gather A (C_in is a multiple of 16, so one K step stays inside one tap) ----
    float4 av = make_float4(0.f, 0.f, 0.f, 0.f);
    if (a_ok) {
      const int tap = k0 / g.C_in;
      const int c = k0 - tap * g.C_in + aq * 4;
      if (AMODE == CT_A_CONV) {
        const int ky = tap / g.KW, kx = tap - ky * g.KW;
        const int iy = aoy * g.stride - g.pad + ky, ix = aox * g.stride - g.pad_w + kx;
        if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W)
          av = Vec4<T>::ld(xb + ((size_t)iy * g.W + ix) * g.ld_in + c);
      } else {
        DcnCorner s;
        if (dcn_corner((float)(aoy - 1 + tap / 3) + om_px[2 * tap], (float)(aox - 1 + tap % 3) + om_px[2 * tap + 1],
                       g.H, g.W, om_px[18 + tap], s)) {
          const int dx = s.dx ? g.ld_in : 0, dy = s.dy ? g.W * g.ld_in : 0;
          const int off[4] = {0, dx, dy, dy + dx};
          const float wq[4] = {s.w00, s.w01, s.w10, s.w11};
          const T* p00 = xb + (s.yc * g.W + s.xc) * g.ld_in + c;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            if (wq[q] != 0.f) {
              const float4 v = Vec4<T>::ld(p00 + off[q]);
              av.x += wq[q] * v.x; av.y += wq[q] * v.y; av.z += wq[q] * v.z; av.w += wq[q] * v.w;
            }
          }
        }
      }
    }
    const float4 bv = __ldg(reinterpret_cast<const float4*>(w + (size_t)(k0 + bk) * ldw + n0 + bo));
    __syncthreads();
    As[aq * 4 + 0][am] = av.x; As[aq * 4 + 1][am] = av.y;
    As[aq * 4 + 2][am] = av.z; As[aq * 4 + 3][am] = av.w;
    *reinterpret_cast<float4*>(&Bs[bk][bo]) = bv;
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[kk][tm * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tn * 4]);
      const float aa[4] = {a.x, a.y, a.z, a.w}, bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(aa[i], bb[j], acc[i][j]);
    }
  }

  // ---- epilogue ----
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int p = m0 + tm * 4 + i;
    if (p >= g.P_out) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int o = n0 + tn * 4 + j;
      if (o >= g.C_out) continue;
      float v = acc[i][j] + (shift ? shift[o] : 0.f);
      if (residual) v += Elem<T>::ld(residual + (size_t)p * g.ld_res + o);
      if (g.relu) v = fmaxf(v, 0.f);
      if (g.out_mode == CT_OUT_NHWC) {
        Elem<T>::st(reinterpret_cast<T*>(out) + (size_t)p * g.ld_out + o, v);
      } else if (g.out_mode == CT_OUT_NHWC_F32) {
        if (o >= g.sig_from) v = sigmoidf_ref(v);
        reinterpret_cast<float*>(out)[(size_t)p * g.ld_out + o] = v;
      } else {
        const int hw = g.OH * g.OW;
        const int b = p / hw, r = p - b * hw;
        reinterpret_cast<float*>(out)[((size_t)b * g.C_out + o) * hw + r] =
            head_transform(v, g.head_act, g.depth_scale);
      }
    }
  }
}

template <typename T>
static int launch_simt(const ct_conv_desc* d, const ConvGeom& g, cudaStream_t st) {
  const int ldw = (g.C_out + 63) / 64 * 64;
  dim3 grid((g.P_out + BM - 1) / BM, ldw / BN);
  if (d->a_mode == CT_A_DCN)
    conv_simt_kernel<T, CT_A_DCN><<<grid, NT, 0, st>>>(
        g, (const T*)d->x, (const float*)d->w, ldw, d->shift, (const T*)d->residual, d->om, d->out);
  else
    conv_simt_kernel<T, CT_A_CONV><<<grid, NT, 0, st>>>(
        g, (const T*)d->x, (const float*)d->w, ldw, d->shift, (const T*)d->residual, d->om, d->out);
  return after_launch();
}

// No dynamic shared memory and no pipeline: the configuration stays all zero.
int conv_config_simt(const ct_conv_desc* d, ConvConfig* c) {
  if (d->C_in % 16 != 0) return fail(CT_ERR_INVALID, "conv_simt: C_in must be a multiple of 16%s (%ld)", "", d->C_in);
  if (d->ld_in % 4 != 0) return fail(CT_ERR_INVALID, "conv_simt: ld_in %% 4 != 0%s", "");
  *c = ConvConfig{};
  return CT_OK;
}

int conv_forward_simt(const ct_conv_desc* d, cudaStream_t st) {
  ConvConfig c;
  const int rc = conv_config_simt(d, &c);
  if (rc != CT_OK) return rc;
  const ConvGeom g = make_geom(d);
  return d->dtype == CT_F32 ? launch_simt<float>(d, g, st) : launch_simt<__nv_bfloat16>(d, g, st);
}

}  // namespace ctb
