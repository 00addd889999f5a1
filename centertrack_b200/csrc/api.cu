// C-ABI glue: error state, launch accounting, host-side weight packing, engine dispatch.
#include "conv_common.cuh"
#include <vector>

namespace ctb {
thread_local char g_err[512] = {0};
thread_local int64_t g_launches = 0;

static inline uint16_t f32_to_bf16_rn(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);  // NaN
  const uint32_t lsb = (u >> 16) & 1u;
  u += 0x7fffu + lsb;
  return (uint16_t)(u >> 16);
}
}  // namespace ctb

using namespace ctb;

extern "C" const char* ct_last_error(void) { return g_err; }
extern "C" int ct_abi_version(void) { return CTB200_ABI_VERSION; }
extern "C" int64_t ct_launch_count(void) { return g_launches; }
extern "C" void ct_reset_launch_count(void) { g_launches = 0; }
extern "C" int ct_debug_trace(void* device_buf) {
  const int r = halo_set_trace(device_buf);
  return r != CT_OK ? r : tc_set_trace(device_buf);
}
extern "C" int ct_debug_watch(void* mapped_host_buf) {
  int r = halo_set_watch(mapped_host_buf);
  if (r == CT_OK) r = tc_set_watch(mapped_host_buf);
  if (r == CT_OK) r = decode_set_watch(mapped_host_buf);
  return r;
}

static inline int tc_k_slices(int C_in, int KH, int KW) { return (KH * KW * C_in + 63) / 64; }

extern "C" int64_t ct_packed_weight_bytes(int32_t engine, int32_t C_out, int32_t C_in, int32_t KH,
                                          int32_t KW, int32_t n_tile) {
  if (engine == CT_ENGINE_SIMT) {
    const int64_t ldw = (C_out + 63) / 64 * 64;
    return (int64_t)KH * KW * C_in * ldw * 4;
  }
  if (n_tile <= 0 || n_tile % 16 != 0 || n_tile > 256) return -1;
  const int64_t n_tiles = (C_out + n_tile - 1) / n_tile;
  if (engine == CT_ENGINE_TCGEN05_HALO) {
    if (!(C_in == 8 || (C_in % 16 == 0 && C_in <= 64) || (C_in % 64 == 0 && C_in <= 256))) return -1;
    return n_tiles * halo_blocks(C_in, KH, KW) * (int64_t)n_tile * 32;
  }
  return n_tiles * tc_k_slices(C_in, KH, KW) * (int64_t)n_tile * 64 * 2 * (engine == CT_ENGINE_TCGEN05_X3 ? 2 : 1);
}

extern "C" int ct_pack_weights(int32_t engine, const float* w, int32_t C_out, int32_t C_in, int32_t KH,
                               int32_t KW, int32_t n_tile, void* dst) {
  CT_REQUIRE(w && dst, "null pointer");
  CT_REQUIRE(C_out > 0 && C_in > 0 && KH > 0 && KW > 0, "bad shape");
  const int taps = KH * KW;
  if (engine == CT_ENGINE_SIMT) {
    const int ldw = (C_out + 63) / 64 * 64;
    float* o = (float*)dst;
    memset(o, 0, (size_t)taps * C_in * ldw * 4);
    for (int oc = 0; oc < C_out; ++oc)
      for (int c = 0; c < C_in; ++c)
        for (int t = 0; t < taps; ++t)
          o[((size_t)t * C_in + c) * ldw + oc] = w[((size_t)oc * C_in + c) * taps + t];
    return CT_OK;
  }
  CT_REQUIRE(n_tile > 0 && n_tile % 16 == 0 && n_tile <= 256, "bad n_tile");
  CT_REQUIRE(C_in % 8 == 0, "C_in must be a multiple of 8 for the wgmma engines");
  if (engine == CT_ENGINE_TCGEN05_HALO) {
    CT_REQUIRE(C_in == 8 || (C_in % 16 == 0 && C_in <= 64) || (C_in % 64 == 0 && C_in <= 256),
               "halo engine: C_in in {8,16,32,48,64,128,192,256}");
    const int nblk = halo_blocks(C_in, KH, KW), n_tiles = (C_out + n_tile - 1) / n_tile, groups = n_tile / 8;
    uint16_t* o = (uint16_t*)dst;
    memset(o, 0, (size_t)n_tiles * nblk * n_tile * 32);
    const int pairs = (KW + 1) / 2;
    for (int oc = 0; oc < C_out; ++oc) {
      const int nt = oc / n_tile, r = oc % n_tile, grp = r / 8, row = r % 8;
      for (int ky = 0; ky < KH; ++ky)
        for (int kx = 0; kx < KW; ++kx)
          for (int c = 0; c < C_in; ++c) {
            int blk, kc, e;
            if (C_in == 8) { blk = ky * pairs + kx / 2; kc = kx & 1; e = c; }
            else { blk = (ky * KW + kx) * (C_in / 16) + c / 16; kc = (c % 16) / 8; e = c % 8; }
            const size_t off = ((((size_t)nt * nblk + blk) * 2 + kc) * groups + grp) * 64 + row * 8 + e;
            o[off] = f32_to_bf16_rn(w[((size_t)oc * C_in + c) * taps + ky * KW + kx]);
          }
    }
    return CT_OK;
  }
  const int ks = tc_k_slices(C_in, KH, KW);
  const int n_tiles = (C_out + n_tile - 1) / n_tile;
  const int parts = engine == CT_ENGINE_TCGEN05_X3 ? 2 : 1;     // x3: [hi tile][lo tile] per K slice
  uint16_t* o = (uint16_t*)dst;
  memset(o, 0, (size_t)n_tiles * ks * n_tile * 64 * 2 * parts);
  for (int oc = 0; oc < C_out; ++oc) {
    const int nt = oc / n_tile, r = oc % n_tile;
    for (int t = 0; t < taps; ++t)
      for (int c = 0; c < C_in; ++c) {
        const int k = t * C_in + c;
        const int s = k / 64, j = k % 64;
        const int chunk = (j / 8) ^ (r & 7);           // 128B swizzle: 16B chunk index XOR row%8
        const size_t off = ((size_t)nt * ks + s) * n_tile * 64 * parts + (size_t)r * 64 + chunk * 8 + (j % 8);
        const float wv = w[((size_t)oc * C_in + c) * taps + t];
        const uint16_t hi = f32_to_bf16_rn(wv);
        o[off] = hi;
        if (parts == 2) {
          uint32_t hu = (uint32_t)hi << 16;
          float hf;
          memcpy(&hf, &hu, 4);
          o[off + (size_t)n_tile * 64] = f32_to_bf16_rn(wv - hf);
        }
      }
  }
  return CT_OK;
}

// The checks every engine shares; each engine's configuration step adds its own.  No pointer is looked at: both
// ct_conv_config and ct_conv_forward run this.
static int check_conv_desc(const ct_conv_desc* d) {
  CT_REQUIRE(d->B > 0 && d->H > 0 && d->W > 0 && d->C_in > 0 && d->C_out > 0, "bad shape");
  // `pad` is the top / left padding; fewer output rows / columns than the symmetric count mean less padding at the
  // bottom / right (even kernels: 2x2, pad 1 -> taps {-1, 0}, OH = H).  Accepted by the halo engine only.
  const int oh_full = (d->H + 2 * d->pad - d->KH) / d->stride + 1;
  CT_REQUIRE(d->OH == oh_full || (d->engine == CT_ENGINE_TCGEN05_HALO && d->OH >= 1 && d->OH < oh_full), "OH inconsistent");
  {
    const int pad_w = d->pad_w1 > 0 ? d->pad_w1 - 1 : d->pad;
    const int ow_full = (d->W + 2 * pad_w - d->KW) / d->stride + 1;
    CT_REQUIRE(d->OW == ow_full || (d->engine == CT_ENGINE_TCGEN05_HALO && d->OW >= 1 && d->OW < ow_full), "OW inconsistent");
    CT_REQUIRE(d->pad_w1 == 0 || d->engine != CT_ENGINE_TCGEN05_HALO, "halo engine: square 'same' kernels only");
  }
  CT_REQUIRE(d->ld_in >= d->C_in, "ld_in < C_in");
  CT_REQUIRE(d->out_mode == CT_OUT_NCHW_F32 || d->ld_out >= (d->epilogue_sum3 ? 16 : d->C_out), "ld_out < C_out");
  if (d->a_mode == CT_A_DCN || d->a_mode == CT_A_DCN_WIN) {
    CT_REQUIRE(d->ld_om >= 27, "DCN needs om with ld_om >= 27");
    CT_REQUIRE(d->a_mode == CT_A_DCN || d->engine == CT_ENGINE_TCGEN05, "CT_A_DCN_WIN: bf16 wgmma engine only");
    CT_REQUIRE(d->KH == 3 && d->KW == 3 && d->stride == 1 && d->pad == 1, "DCN is 3x3 s1 p1");
  }
  CT_REQUIRE(d->out_mode != CT_OUT_NHWC_S2D || d->engine == CT_ENGINE_TCGEN05_HALO, "CT_OUT_NHWC_S2D: halo engine only");
  switch (d->engine) {
    case CT_ENGINE_SIMT:
      return CT_OK;
    case CT_ENGINE_TCGEN05:
      CT_REQUIRE(d->dtype == CT_BF16, "wgmma engine needs bf16 activations");
      return CT_OK;
    case CT_ENGINE_TCGEN05_X3:
      CT_REQUIRE(d->dtype == CT_F32, "wgmma x3 engine runs on fp32 activations");
      return CT_OK;
    case CT_ENGINE_TCGEN05_HALO:
      CT_REQUIRE(d->dtype == CT_BF16 && d->a_mode == CT_A_CONV, "halo engine: bf16 plain convolutions");
      return CT_OK;
    default:
      return fail(CT_ERR_INVALID, "unknown engine%s %ld", "", (long)d->engine);
  }
}

extern "C" int ct_conv_config(const ct_conv_desc* d, struct ct_conv_config* out) {
  CT_REQUIRE(d && out, "null pointer");
  const int r = check_conv_desc(d);
  if (r != CT_OK) return r;
  *out = ConvConfig{};
  if (d->engine == CT_ENGINE_SIMT) return conv_config_simt(d, out);
  if (d->engine == CT_ENGINE_TCGEN05_HALO) return d->n_heads ? conv_config_heads(d, out) : conv_config_halo(d, out);
  return conv_config_tc(d, out);
}

extern "C" int ct_conv_forward(const ct_conv_desc* d, void* stream) {
  CT_REQUIRE(d && d->x && d->w && (d->out || d->n_heads), "null pointer");
  CT_REQUIRE(d->om || (d->a_mode != CT_A_DCN && d->a_mode != CT_A_DCN_WIN), "DCN needs om with ld_om >= 27");
  const int r = check_conv_desc(d);
  if (r != CT_OK) return r;
  cudaStream_t st = (cudaStream_t)stream;
  if (d->engine == CT_ENGINE_SIMT) return conv_forward_simt(d, st);
  if (d->engine == CT_ENGINE_TCGEN05_HALO) return d->n_heads ? conv_forward_heads(d, st) : conv_forward_halo(d, st);
  return conv_forward_tc(d, st);
}
