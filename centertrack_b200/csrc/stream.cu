// Per-stream state kept on the device between frames (SURVEY 8f rows 1-3):
//   ct_track_step    generic_post_process's affine + Tracker.step's greedy displacement association
//                    (utils/post_process.py:21-91, utils/tracker.py:28-138) on the packed decode records, plus the
//                    (centre, radius) boxes of Detector._get_additional_inputs (detector.py:254-290) for the NEXT frame
//   ct_render_tracks the gaussian max-splat of those boxes into pre_hm (image.py:128-154)
//   ct_flip_merge    Detector._flip_output (detector.py:311-332; model/utils.py:28-50) for --flip_test
//   ct_warp_affine_normalize   Detector.pre_process's cv2.warpAffine(INTER_LINEAR) + (x/255 - mean)/std + HWC->CHW
//                    (detector.py:207-226), cv2's fixed-point bilinear restated
// All HBM-bound byte/index work: one pass over the data, coalesced, no tensor cores.
#include "common.cuh"

namespace ctb {

// ------------------------------------------------------------------------------------------------------------------
// flip merge: out[c,y,x] = 0.5 * (in[0,c,y,x] + sign[c] * in[1,perm[c],y,W-1-x])
// ------------------------------------------------------------------------------------------------------------------
__global__ void flip_merge_kernel(const float* __restrict__ in2, float* __restrict__ out, int C, int H, int W,
                                  const int* __restrict__ perm, const float* __restrict__ sign) {
  const size_t total = (size_t)C * H * W;
  const size_t plane = (size_t)H * W;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i / plane);
    const size_t r = i - (size_t)c * plane;
    const int y = (int)(r / W), x = (int)(r - (size_t)y * W);
    const int cs = perm ? perm[c] : c;
    const float sg = sign ? sign[c] : 1.f;
    const float a = in2[i];
    const float b = in2[total + (size_t)cs * plane + (size_t)y * W + (W - 1 - x)];
    // the reference adds the two maps and halves the sum: (a + s*b) / 2, in that order (division by 2 is exact)
    out[i] = __fmul_rn(__fadd_rn(a, __fmul_rn(sg, b)), 0.5f);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// track step
// ------------------------------------------------------------------------------------------------------------------
constexpr int TRK_THREADS = 128;
constexpr int TF = CT_TRK_FLOATS;

struct TrackArgs {
  ct_track_desc d;
};

__device__ __forceinline__ float aff_f32(const float* t, float x, float y) {
  // np.dot(trans[2x3] f32, [x, y, 1] f32): x*t0 + y*t1 + t2 accumulated left to right in fp32
  return __fadd_rn(__fadd_rn(__fmul_rn(t[0], x), __fmul_rn(t[1], y)), t[2]);
}
__device__ __forceinline__ double aff_f64(const double* t, double x, double y) {
  return __dadd_rn(__dadd_rn(__dmul_rn(t[0], x), __dmul_rn(t[1], y)), t[2]);
}

// gaussian_radius(det_size=(h, w), min_overlap=0.7): utils/image.py:105-125, float64
__device__ double gaussian_radius_f64(double h, double w) {
  const double mo = 0.7;
  const double b1 = h + w;
  const double c1 = w * h * (1 - mo) / (1 + mo);
  const double r1 = (b1 + sqrt(b1 * b1 - 4 * c1)) / 2;
  const double b2 = 2 * (h + w);
  const double c2 = (1 - mo) * w * h;
  const double r2 = (b2 + sqrt(b2 * b2 - 16 * c2)) / 2;
  const double a3 = 4 * mo;
  const double b3 = -2 * mo * (h + w);
  const double c3 = (mo - 1) * w * h;
  const double r3 = (b3 + sqrt(b3 * b3 - 4 * a3 * c3)) / 2;
  return fmin(r1, fmin(r2, r3));
}

__global__ void __launch_bounds__(TRK_THREADS)
track_step_kernel(const TrackArgs a) {
  extern __shared__ __align__(16) unsigned char tsm[];
  const ct_track_desc& d = a.d;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int T = d.max_tracks, K = d.K;
  float* s_old = reinterpret_cast<float*>(tsm);                 // [T][TF]   previous tracks
  float* s_det = s_old + (size_t)T * TF;                        // [K][TF]   this frame's detections (image coords)
  float* s_px = s_det + (size_t)K * TF;                         // [K] predicted previous centre x (ct + tracking)
  float* s_py = s_px + K;                                       // [K]
  float* s_isz = s_py + K;                                      // [K] detection box area
  float* s_tsz = s_isz + K;                                     // [T] track box area
  int* s_match = reinterpret_cast<int*>(s_tsz + T);             // [K] matched track or -1
  int* s_taken = s_match + K;                                   // [T]
  int* s_pos_det = s_taken + T;                                 // [K] output slot of det or -1
  int* s_pos_trk = s_pos_det + K;                               // [T] output slot of a coasting track or -1
  __shared__ float red_v[TRK_THREADS / 32];
  __shared__ int red_j[TRK_THREADS / 32];
  __shared__ int s_n, s_total, s_ids;

  int M = d.counts[b * 2 + 0];
  if (M > T) M = T;
  const int id_count = d.counts[b * 2 + 1];
  float* trk = d.tracks + (size_t)b * T * TF;
  for (int i = tid; i < M * TF; i += TRK_THREADS) s_old[i] = trk[i];
  if (tid == 0) s_n = 0;
  __syncthreads();

  // ---- detections of this frame: generic_post_process (post_process.py:21-91), merge_outputs (detector.py:371-377)
  const float* rec = d.records + (size_t)b * K * d.F;
  const float* to = d.trans_out_inv + b * 6;
  int cnt = 0;
  for (int i = tid; i < K; i += TRK_THREADS) cnt += rec[(size_t)i * d.F + CT_REC_SCORE] > d.out_thresh ? 1 : 0;
  atomicAdd(&s_n, cnt);
  __syncthreads();
  const int N = s_n;                     // records are sorted by score: the kept detections are a prefix
  for (int i = tid; i < N; i += TRK_THREADS) {
    const float* r = rec + (size_t)i * d.F;
    float* o = s_det + (size_t)i * TF;
    const float cx = r[CT_REC_XS], cy = r[CT_REC_YS];
    const float ctx = aff_f32(to, cx, cy), cty = aff_f32(to + 3, cx, cy);
    float tx = 0.f, ty = 0.f;
    if (d.rec_tracking >= 0) {
      const float px = __fadd_rn(r[d.rec_tracking], cx), py = __fadd_rn(r[d.rec_tracking + 1], cy);
      tx = __fsub_rn(aff_f32(to, px, py), ctx);
      ty = __fsub_rn(aff_f32(to + 3, px, py), cty);
    }
    const float bl = r[CT_REC_BBOX], bt = r[CT_REC_BBOX + 1], br = r[CT_REC_BBOX + 2], bb = r[CT_REC_BBOX + 3];
    o[CT_TRK_SCORE] = r[CT_REC_SCORE];
    o[CT_TRK_CLASS] = r[CT_REC_CLS] + 1.f;
    o[CT_TRK_CT] = ctx; o[CT_TRK_CT + 1] = cty;
    o[CT_TRK_TRACKING] = tx; o[CT_TRK_TRACKING + 1] = ty;
    o[CT_TRK_BBOX] = aff_f32(to, bl, bt); o[CT_TRK_BBOX + 1] = aff_f32(to + 3, bl, bt);
    o[CT_TRK_BBOX + 2] = aff_f32(to, br, bb); o[CT_TRK_BBOX + 3] = aff_f32(to + 3, br, bb);
    o[CT_TRK_ID] = 0.f; o[CT_TRK_AGE] = 1.f; o[CT_TRK_ACTIVE] = 0.f;
    s_px[i] = __fadd_rn(ctx, tx);
    s_py[i] = __fadd_rn(cty, ty);
    s_isz[i] = __fmul_rn(__fsub_rn(o[CT_TRK_BBOX + 2], o[CT_TRK_BBOX]), __fsub_rn(o[CT_TRK_BBOX + 3], o[CT_TRK_BBOX + 1]));
    s_match[i] = -1;
  }
  for (int j = tid; j < M; j += TRK_THREADS) {
    const float* t = s_old + (size_t)j * TF;
    s_tsz[j] = __fmul_rn(__fsub_rn(t[CT_TRK_BBOX + 2], t[CT_TRK_BBOX]), __fsub_rn(t[CT_TRK_BBOX + 3], t[CT_TRK_BBOX + 1]));
    s_taken[j] = 0;
  }
  __syncthreads();

  // ---- greedy assignment (tracker.py:129-138): detections in score order take their nearest free, valid track;
  //      argmin ties -> lowest track index
  const float INF = 3.0e38f;
  for (int i = 0; i < N && M > 0; ++i) {
    const float px = s_px[i], py = s_py[i], isz = s_isz[i], icls = s_det[(size_t)i * TF + CT_TRK_CLASS];
    float best = INF;
    int bj = 0x7fffffff;
    for (int j = tid; j < M; j += TRK_THREADS) {
      const float* t = s_old + (size_t)j * TF;
      const float dx = __fsub_rn(t[CT_TRK_CT], px), dy = __fsub_rn(t[CT_TRK_CT + 1], py);
      const float dist = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
      const bool ok = !s_taken[j] && !(dist > s_tsz[j]) && !(dist > isz) && t[CT_TRK_CLASS] == icls;
      if (ok && dist < best) { best = dist; bj = j; }       // ascending j per thread: first minimum kept
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (ov < best || (ov == best && oj < bj)) { best = ov; bj = oj; }
    }
    if (lane == 0) { red_v[warp] = best; red_j[warp] = bj; }
    __syncthreads();
    if (tid == 0) {
      float v = red_v[0];
      int j = red_j[0];
      for (int w = 1; w < TRK_THREADS / 32; ++w)
        if (red_v[w] < v || (red_v[w] == v && red_j[w] < j)) { v = red_v[w]; j = red_j[w]; }
      if (v < 1e16f && j < M) { s_match[i] = j; s_taken[j] = 1; }
    }
    __syncthreads();
  }

  // ---- output order (tracker.py:74-127): matched detections, then new tracks, then coasting tracks
  if (tid == 0) {
    int pos = 0, ids = id_count;
    for (int i = 0; i < N; ++i) {
      s_pos_det[i] = -1;
      if (s_match[i] >= 0) {
        float* o = s_det + (size_t)i * TF;
        const float* t = s_old + (size_t)s_match[i] * TF;
        o[CT_TRK_ID] = t[CT_TRK_ID]; o[CT_TRK_AGE] = 1.f; o[CT_TRK_ACTIVE] = t[CT_TRK_ACTIVE] + 1.f;
        if (pos < T) s_pos_det[i] = pos++;
      }
    }
    for (int i = 0; i < N; ++i) {
      if (s_match[i] >= 0) continue;
      float* o = s_det + (size_t)i * TF;
      if (o[CT_TRK_SCORE] > d.new_thresh) {
        ++ids;
        o[CT_TRK_ID] = (float)ids; o[CT_TRK_AGE] = 1.f; o[CT_TRK_ACTIVE] = 1.f;
        if (pos < T) s_pos_det[i] = pos++;
      }
    }
    for (int j = 0; j < M; ++j) {
      s_pos_trk[j] = -1;
      if (s_taken[j]) continue;
      float* t = s_old + (size_t)j * TF;
      if (t[CT_TRK_AGE] < (float)d.max_age) {
        t[CT_TRK_AGE] += 1.f; t[CT_TRK_ACTIVE] = 0.f;
        if (pos < T) s_pos_trk[j] = pos++;
      }
    }
    s_total = pos;
    s_ids = ids;
  }
  __syncthreads();
  const int total = s_total;
  for (int e = tid; e < N * TF; e += TRK_THREADS) {
    const int i = e / TF, f = e - i * TF;
    if (s_pos_det[i] >= 0) trk[(size_t)s_pos_det[i] * TF + f] = s_det[e];
  }
  for (int e = tid; e < M * TF; e += TRK_THREADS) {
    const int j = e / TF, f = e - j * TF;
    if (s_pos_trk[j] >= 0) trk[(size_t)s_pos_trk[j] * TF + f] = s_old[e];
  }
  if (tid == 0) { d.counts[b * 2 + 0] = total; d.counts[b * 2 + 1] = s_ids; }
  __syncthreads();     // the table rows written above are re-read below by other threads
  __threadfence_block();

  // ---- boxes of the NEXT frame's prior heat-map (detector.py:254-290): image -> input coords, clip, radius, centre
  if (d.boxes) {
    const double* ti = d.trans_input + b * 6;
    float* bx = d.boxes + (size_t)b * T * 5;
    for (int r = tid; r < T; r += TRK_THREADS) {
      float radius = -1.f, cxo = 0.f, cyo = 0.f;
      if (r < total) {
        const float* t = trk + (size_t)r * TF;
        if (!(t[CT_TRK_SCORE] < d.pre_thresh) && t[CT_TRK_ACTIVE] != 0.f) {
          const float wmax = (float)(d.inp_w - 1), hmax = (float)(d.inp_h - 1);
          float x0 = (float)aff_f64(ti, (double)t[CT_TRK_BBOX], (double)t[CT_TRK_BBOX + 1]);
          float y0 = (float)aff_f64(ti + 3, (double)t[CT_TRK_BBOX], (double)t[CT_TRK_BBOX + 1]);
          float x1 = (float)aff_f64(ti, (double)t[CT_TRK_BBOX + 2], (double)t[CT_TRK_BBOX + 3]);
          float y1 = (float)aff_f64(ti + 3, (double)t[CT_TRK_BBOX + 2], (double)t[CT_TRK_BBOX + 3]);
          x0 = fminf(fmaxf(x0, 0.f), wmax); x1 = fminf(fmaxf(x1, 0.f), wmax);
          y0 = fminf(fmaxf(y0, 0.f), hmax); y1 = fminf(fmaxf(y1, 0.f), hmax);
          const float h = __fsub_rn(y1, y0), w = __fsub_rn(x1, x0);
          if (h > 0.f && w > 0.f) {
            const double rad = gaussian_radius_f64(ceil((double)h), ceil((double)w));
            const int ri = (int)rad;                 // int(): truncation
            radius = (float)(ri > 0 ? ri : 0);
            cxo = (float)(int)(__fadd_rn(x0, x1) * 0.5f);   // astype(np.int32): truncation
            cyo = (float)(int)(__fadd_rn(y0, y1) * 0.5f);
          }
        }
      }
      bx[r * 5 + 0] = (float)b; bx[r * 5 + 1] = cxo; bx[r * 5 + 2] = cyo; bx[r * 5 + 3] = radius; bx[r * 5 + 4] = 0.f;
    }
  }
}

// splat of the boxes written by track_step_kernel; rows with radius < 0 are skipped.  grid = B*T (fixed: graph-capturable)
__global__ void render_tracks_kernel(const float* __restrict__ boxes, int n, float* __restrict__ hm, int B, int H, int W) {
  const int i = blockIdx.x;
  if (i >= n) return;
  const float rf = boxes[i * 5 + 3];
  if (rf < 0.f) return;
  const int b = (int)boxes[i * 5 + 0], cx = (int)boxes[i * 5 + 1], cy = (int)boxes[i * 5 + 2], r = (int)rf;
  if (b < 0 || b >= B) return;
  const double sigma = (double)(2 * r + 1) / 6.0;
  const int left = min(cx, r), right = min(W - cx, r + 1), top = min(cy, r), bottom = min(H - cy, r + 1);
  const int w = left + right, h = top + bottom;
  if (w <= 0 || h <= 0) return;
  for (int j = threadIdx.x; j < w * h; j += blockDim.x) {
    const int yy = j / w - top, xx = j % w - left;
    double v = exp(-(double)(xx * xx + yy * yy) / (2.0 * sigma * sigma));
    if (v < 2.220446049250313e-16) v = 0.0;
    atomicMax(reinterpret_cast<int*>(hm + ((size_t)b * H + cy + yy) * W + cx + xx), __float_as_int((float)v));
  }
}

// ------------------------------------------------------------------------------------------------------------------
// pre_process: cv2.warpAffine(src u8 HWC, M, (ow, oh), INTER_LINEAR, BORDER_CONSTANT 0) then (v/255 - mean)/std, CHW.
// cv2's arithmetic (imgwarp.cpp warpAffine + remapBilinear): source coordinates in 1/1024 px fixed point rounded
// to 1/32 px, bilinear weights from a 32x32 table of int16 coefficients summing to 2^15, result (sum + 2^14) >> 15.
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int sat_int(double v) {        // cv::saturate_cast<int>(double) = cvRound, ties to even
  return __double2int_rn(v);
}

__global__ void warp_affine_norm_kernel(const unsigned char* __restrict__ src, int sh, int sw, int sstep,
                                        float* __restrict__ dst, int B, int oh, int ow,
                                        const double* __restrict__ minv /*[B][6] dst->src*/, float3 mean, float3 stdv) {
  const size_t total = (size_t)B * oh * ow;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / ((size_t)oh * ow));
    const size_t r = i - (size_t)b * oh * ow;
    const int y = (int)(r / ow), x = (int)(r - (size_t)y * ow);
    const double* M = minv + b * 6;
    const int AB_BITS = 10, AB_SCALE = 1 << AB_BITS, INTER_BITS = 5, INTER_TAB = 1 << INTER_BITS;
    const int round_delta = AB_SCALE / INTER_TAB / 2;
    const int adelta = sat_int(M[0] * x * AB_SCALE), bdelta = sat_int(M[3] * x * AB_SCALE);
    const int X0 = sat_int((M[1] * y + M[2]) * AB_SCALE) + round_delta;
    const int Y0 = sat_int((M[4] * y + M[5]) * AB_SCALE) + round_delta;
    const int X = (X0 + adelta) >> (AB_BITS - INTER_BITS), Y = (Y0 + bdelta) >> (AB_BITS - INTER_BITS);
    const int sx = X >> INTER_BITS, sy = Y >> INTER_BITS;          // arithmetic shifts: floor
    // BilinearTab_i: (1-fy|fy) x (1-fx|fx) in 1/32 steps, scaled by 2^15: exact integers (the table's one saturated
    // entry, fx = fy = 0, yields the same pixel as the exact weight 32768)
    const int fx = X & (INTER_TAB - 1), fy = Y & (INTER_TAB - 1);
    const int w[4] = {(32 - fy) * (32 - fx) * 32, (32 - fy) * fx * 32, fy * (32 - fx) * 32, fy * fx * 32};
    const unsigned char* img = src + (size_t)b * sh * sstep;
    float out[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      int acc = 0;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int yy = sy + (t >> 1), xx = sx + (t & 1);
        const int v = ((unsigned)yy < (unsigned)sh && (unsigned)xx < (unsigned)sw) ? img[(size_t)yy * sstep + xx * 3 + c] : 0;
        acc += v * w[t];
      }
      const int pix = (acc + (1 << 14)) >> 15;
      const int p8 = pix < 0 ? 0 : (pix > 255 ? 255 : pix);
      // ((inp / 255. - mean) / std).astype(float32): float64 arithmetic, one final rounding
      out[c] = (float)p8;
    }
    const size_t plane = (size_t)oh * ow;
    float* o = dst + (size_t)b * 3 * plane + (size_t)y * ow + x;
    o[0] = (float)(((double)out[0] / 255.0 - (double)mean.x) / (double)stdv.x);
    o[plane] = (float)(((double)out[1] / 255.0 - (double)mean.y) / (double)stdv.y);
    o[2 * plane] = (float)(((double)out[2] / 255.0 - (double)mean.z) / (double)stdv.z);
  }
}

}  // namespace ctb

using namespace ctb;

static inline int sw_blocks(size_t total) {
  size_t b = (total + 255) / 256;
  const size_t cap = (size_t)device_sm_count() * 16;
  return (int)(b < cap ? (b ? b : 1) : cap);
}

extern "C" int ct_flip_merge(const float* in2, float* out, int32_t C, int32_t H, int32_t W, const int32_t* perm,
                             const float* sign, void* stream) {
  CT_REQUIRE(in2 && out, "null pointer");
  CT_REQUIRE(C > 0 && H > 0 && W > 0, "bad shape");
  flip_merge_kernel<<<sw_blocks((size_t)C * H * W), 256, 0, (cudaStream_t)stream>>>(in2, out, C, H, W, perm, sign);
  return after_launch();
}

extern "C" int64_t ct_track_smem_bytes(int32_t K, int32_t max_tracks) {
  return (int64_t)((size_t)max_tracks * TF + (size_t)K * TF + 3 * (size_t)K + max_tracks) * 4 +
         (int64_t)(2 * (size_t)K + 2 * (size_t)max_tracks) * 4 + 64;
}

extern "C" int ct_track_step(const ct_track_desc* d, void* stream) {
  CT_REQUIRE(d && d->records && d->trans_out_inv && d->tracks && d->counts, "null pointer");
  CT_REQUIRE(d->B > 0 && d->K > 0 && d->F >= CT_REC_HEADS && d->max_tracks >= d->K, "bad shape");
  CT_REQUIRE(d->rec_tracking < 0 || d->rec_tracking + 2 <= d->F, "tracking offset outside the record");
  CT_REQUIRE(d->boxes == nullptr || (d->trans_input != nullptr && d->inp_h > 0 && d->inp_w > 0), "boxes need trans_input");
  const size_t smem = (size_t)ct_track_smem_bytes(d->K, d->max_tracks);
  CT_REQUIRE(smem <= 200 * 1024, "track table does not fit in shared memory (lower max_tracks)");
  if (smem > 48 * 1024)
    CT_CUDA_OK(cudaFuncSetAttribute(track_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  TrackArgs a;
  a.d = *d;
  track_step_kernel<<<d->B, TRK_THREADS, smem, (cudaStream_t)stream>>>(a);
  return after_launch();
}

extern "C" int ct_render_tracks(const float* boxes, int32_t n, float* pre_hm, int32_t B, int32_t H, int32_t W,
                                void* stream) {
  CT_REQUIRE(pre_hm && boxes && n > 0, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  CT_CUDA_OK(cudaMemsetAsync(pre_hm, 0, (size_t)B * H * W * sizeof(float), st));
  render_tracks_kernel<<<n, 128, 0, st>>>(boxes, n, pre_hm, B, H, W);
  return after_launch();
}

extern "C" int ct_warp_affine_normalize(const uint8_t* src, int32_t B, int32_t src_h, int32_t src_w, int32_t src_step,
                                        const double* minv, const float* mean, const float* std,
                                        float* dst, int32_t out_h, int32_t out_w, void* stream) {
  CT_REQUIRE(src && minv && mean && std && dst, "null pointer");
  CT_REQUIRE(B > 0 && src_h > 0 && src_w > 0 && src_step >= 3 * src_w && out_h > 0 && out_w > 0, "bad shape");
  warp_affine_norm_kernel<<<sw_blocks((size_t)B * out_h * out_w), 256, 0, (cudaStream_t)stream>>>(
      src, src_h, src_w, src_step, dst, B, out_h, out_w, minv, make_float3(mean[0], mean[1], mean[2]),
      make_float3(std[0], std[1], std[2]));
  return after_launch();
}
