// Pieces shared by the SIMT (fp32-exact) and wgmma (bf16) implicit-GEMM engines: output-pixel decomposition, conv
// window addressing and DCNv2 bilinear sampling, and the host-side tensor-map / launch helpers of the wgmma engines.
#pragma once
#include "common.cuh"
#include <cudaTypedefs.h>
#include <type_traits>

namespace ctb {

struct ConvGeom {
  int B, H, W, C_in, ld_in;
  int C_out, KH, KW, stride, pad, pad_w, OH, OW;
  int ld_out, out_mode, relu, ld_res, head_act, sig_from;
  float depth_scale;
  int ld_om;
  int P_out;      // B*OH*OW
  int K_total;    // KH*KW*C_in
};

inline ConvGeom make_geom(const ct_conv_desc* d) {
  ConvGeom g;
  g.B = d->B; g.H = d->H; g.W = d->W; g.C_in = d->C_in; g.ld_in = d->ld_in;
  g.C_out = d->C_out; g.KH = d->KH; g.KW = d->KW; g.stride = d->stride; g.pad = d->pad;
  g.pad_w = d->pad_w1 > 0 ? d->pad_w1 - 1 : d->pad;
  g.OH = d->OH; g.OW = d->OW; g.ld_out = d->ld_out; g.out_mode = d->out_mode;
  g.relu = d->relu; g.ld_res = d->ld_res; g.head_act = d->head_act; g.sig_from = d->sig_from;
  g.depth_scale = d->depth_scale; g.ld_om = d->ld_om;
  g.P_out = d->B * d->OH * d->OW;
  g.K_total = d->KH * d->KW * d->C_in;
  return g;
}

// Modulated-deformable sampling of one (output pixel, tap):  SURVEY.md Appendix B.
//   py = y - 1 + i + dy_k,  px = x - 1 + j + dx_k ;  S = 0 unless -1 < py < H and -1 < px < W ;
//   bilinear over the integer neighbours that lie inside the image; the whole sample times mask.
// dcn_corner gives the footprint of (py, px) in an H x W image, from which every engine samples: top-left corner
// (y0, x0) and its clamp into the image (yc, xc), whether the x+1 / y+1 neighbours exist on both sides (dx, dy), and
// the four corner weights times the mask, zero for corners outside the image.  A corner of non-zero weight is the
// pixel (yc, xc) stepped by dy / dx where it lies below / right of the top-left one.  Returns false (c untouched)
// when the sample is outside the image altogether (its value is 0).
struct DcnCorner { int y0, x0, yc, xc; bool dx, dy; float w00, w01, w10, w11; };
__device__ __forceinline__ bool dcn_corner(float py, float px, int H, int W, float m, DcnCorner& c) {
  if (!(py > -1.f && py < (float)H && px > -1.f && px < (float)W)) return false;
  const float y0f = floorf(py), x0f = floorf(px);
  const int y0 = (int)y0f, x0 = (int)x0f;
  const float ly = py - y0f, lx = px - x0f, hy = 1.f - ly, hx = 1.f - lx;
  const bool y0ok = y0 >= 0, y1ok = y0 + 1 <= H - 1, x0ok = x0 >= 0, x1ok = x0 + 1 <= W - 1;
  c.y0 = y0; c.x0 = x0; c.yc = max(y0, 0); c.xc = max(x0, 0);
  c.dx = x0ok && x1ok; c.dy = y0ok && y1ok;
  c.w00 = (y0ok && x0ok) ? hy * hx * m : 0.f;
  c.w01 = (y0ok && x1ok) ? hy * lx * m : 0.f;
  c.w10 = (y1ok && x0ok) ? ly * hx * m : 0.f;
  c.w11 = (y1ok && x1ok) ? ly * lx * m : 0.f;
  return true;
}

// Apply the per-channel epilogue transform of fp32 head planes.
__device__ __forceinline__ float head_transform(float v, int head_act, float depth_scale) {
  if (head_act == CT_HEAD_SIGMOID) return sigmoidf_ref(v);
  if (head_act == CT_HEAD_DEPTH) return (1.f / (sigmoidf_ref(v) + 1e-6f) - 1.f) * depth_scale;
  return v;
}

// ---- host side of the tensor-core engines ----
// TMA descriptor of a bf16 tensor: `rank` dims and box sizes innermost first, rank - 1 byte strides of the outer
// dims; elements outside the tensor read as zero.  cuTensorMapEncodeTiled is reached through the runtime's driver
// entry point (no -lcuda at link time).
inline int encode_tmap_bf16(CUtensorMap* map, const void* ptr, int rank, const cuuint64_t* dims,
                            const cuuint64_t* strides, const cuuint32_t* box, CUtensorMapSwizzle swizzle) {
  static const PFN_cuTensorMapEncodeTiled encode = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    const bool ok = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
                    q == cudaDriverEntryPointSuccess;
    return ok ? reinterpret_cast<PFN_cuTensorMapEncodeTiled>(p) : nullptr;
  }();
  if (!encode) return fail(CT_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable%s", "");
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  const CUresult cr = encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), dims,
                             strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return cr == CUDA_SUCCESS ? CT_OK : fail(CT_ERR_CUDA, "cuTensorMapEncodeTiled failed%s (%ld)", "", (long)cr);
}

// Launches Kernel with programmatic dependent launch and up to 227 KB of dynamic shared memory.  That limit is a
// per-device attribute of the kernel: it is set on the first launch on each device (per host thread).
template <auto Kernel, typename... Args>
int launch_big_smem(dim3 grid, dim3 block, size_t smem, cudaStream_t st, const Args&... args) {
  int dev = 0;
  cudaGetDevice(&dev);
  static thread_local unsigned long long attr_set_mask = 0;
  if (dev >= 64 || !((attr_set_mask >> dev) & 1ull)) {
    CT_CUDA_OK(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    if (dev < 64) attr_set_mask |= 1ull << dev;
  }
  CT_CUDA_OK(launch_kernel(Kernel, grid, block, smem, st, true, args...));
  return after_launch();
}

// f(std::integral_constant<int, n_tile>()) for the N tiles the tensor-core kernels are instantiated for: 16, 32, .., 256
template <int N = 16, typename F>
int dispatch_n_tile(int n_tile, F&& f) {
  if constexpr (N > 256) return fail(CT_ERR_INVALID, "unsupported n_tile%s (%ld)", "", (long)n_tile);
  else return n_tile == N ? f(std::integral_constant<int, N>()) : dispatch_n_tile<N + 16>(n_tile, f);
}

typedef struct ct_conv_config ConvConfig;

// Each engine's configuration step (ct_conv_config: its shape checks and launch configuration, no CUDA call) and its
// forward, which runs that step and then launches.
int conv_config_simt(const ct_conv_desc* d, ConvConfig* c);
int conv_config_tc(const ct_conv_desc* d, ConvConfig* c);
int conv_config_halo(const ct_conv_desc* d, ConvConfig* c);
int conv_config_heads(const ct_conv_desc* d, ConvConfig* c);
int conv_forward_simt(const ct_conv_desc* d, cudaStream_t st);
int conv_forward_tc(const ct_conv_desc* d, cudaStream_t st);
int conv_forward_halo(const ct_conv_desc* d, cudaStream_t st);
int conv_forward_heads(const ct_conv_desc* d, cudaStream_t st);
int halo_blocks(int C_in, int KH, int KW);
int halo_set_trace(void* buf);
int tc_set_trace(void* buf);
int halo_set_watch(void* mapped_host_buf);
int tc_set_watch(void* mapped_host_buf);
int decode_set_watch(void* mapped_host_buf);

}  // namespace ctb
