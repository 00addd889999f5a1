// Per-stream state kept on the device between frames (SURVEY 8f rows 1-3):
//   ct_track_step    generic_post_process's affine + Tracker.step's greedy displacement association
//                    (utils/post_process.py:21-91, utils/tracker.py:28-138) on the packed decode records, plus the
//                    (centre, radius) boxes of Detector._get_additional_inputs (detector.py:254-290) for the NEXT frame;
//                    ct_track_step_assoc: the same kernel with --hungarian (scipy's linear_sum_assignment restated,
//                    one warp) and / or --public_det births (tracker.py:52-72,83-103); ct_track_step_payload: also
//                    the pose / 3D / velocity / attribute fields of generic_post_process (post_process.py:55-89) in a
//                    payload table beside the track table, and the amodal centre on 3D head sets
//   ct_render_tracks the gaussian max-splat of those boxes into pre_hm (image.py:128-154)
//   ct_flip_merge    Detector._flip_output (detector.py:311-332; model/utils.py:28-50) for --flip_test;
//                    ct_flip_merge_heads: every averaged head of B (frame, mirror) pairs in one launch
//   ct_mirror_x      the mirrored half of a --flip_test batch (detector.py:225-226,285-286)
//   ct_warp_affine_normalize   Detector.pre_process's cv2.warpAffine(INTER_LINEAR) + (x/255 - mean)/std + HWC->CHW
//                    (detector.py:207-226), cv2's fixed-point bilinear restated
//   ct_pack_stem_frames        the same warp + normalise of B ragged uint8 frames (and of their previous frames),
//                    written straight as the tensor-core stem's packed bf16 input; ct_pack_stem_frames_flip also
//                    writes each stream's mirror image (--flip_test)
// All HBM-bound byte/index work: one pass over the data, coalesced, no tensor cores.
#include <math_constants.h>

#include "common.cuh"

namespace ctb {

// ------------------------------------------------------------------------------------------------------------------
// flip merge of B (frame, mirrored frame) pairs, every averaged head in one launch (blockIdx.y = head):
//   out[b,c,y,x] = 0.5 * (in[b,c,y,x] + sign[c] * in[B+b,perm[c],y,W-1-x])
// The descriptors travel in the kernel parameters, so a captured CUDA graph keeps them.
// ------------------------------------------------------------------------------------------------------------------
struct FlipArgs {
  ct_flip_head h[CT_FLIP_MAX_HEADS];
};

__global__ void flip_merge_kernel(const __grid_constant__ FlipArgs fa, int B, int H, int W) {
  const ct_flip_head& hd = fa.h[blockIdx.y];
  const int C = hd.C;
  const size_t plane = (size_t)H * W;
  const size_t img = (size_t)C * plane;
  const size_t total = (size_t)B * img;
  const float* __restrict__ in = hd.in;
  float* __restrict__ out = hd.out;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / img);
    const size_t q = i - (size_t)b * img;
    const int c = (int)(q / plane);
    const size_t r = q - (size_t)c * plane;
    const int y = (int)(r / W), x = (int)(r - (size_t)y * W);
    const int cs = hd.perm ? hd.perm[c] : c;
    const float sg = hd.sign ? hd.sign[c] : 1.f;
    const float a = in[i];
    const float m = in[(size_t)(B + b) * img + (size_t)cs * plane + (size_t)y * W + (W - 1 - x)];
    // the reference adds the two maps and halves the sum: (a + s*b) / 2, in that order (division by 2 is exact)
    out[i] = __fmul_rn(__fadd_rn(a, __fmul_rn(sg, m)), 0.5f);
  }
}

// dst[i,c,y,x] = src[i,c,y,W-1-x]: the mirrored half of a flip-test batch (images, pre_images, pre_hm)
__global__ void mirror_x_kernel(const float* __restrict__ src, float* __restrict__ dst, size_t rows, int W) {
  const size_t total = rows * W;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t row = i / W;
    const int x = (int)(i - row * W);
    dst[i] = src[row * W + (W - 1 - x)];
  }
}

// ------------------------------------------------------------------------------------------------------------------
// track step
// ------------------------------------------------------------------------------------------------------------------
constexpr int TRK_THREADS = 128;
constexpr int TF = CT_TRK_FLOATS;

struct TrackArgs {
  ct_track_desc d;
  ct_track_assoc as;       // all zero: greedy association, private births (ct_track_step)
  ct_track_payload p;      // read by the payload instantiation only
  int pay_smem;            // byte offset of the staged payload rows in dynamic shared memory
};

// bytes of the greedy layout before the association scratch (a multiple of 8: the scratch starts with fp64 arrays)
__host__ __device__ constexpr size_t trk_base_bytes(size_t K, size_t T) { return (16 * T + 18 * K) * 4; }

// Sort key of one column in a Dijkstra step of the assignment solver: the lowest shortest-path cost wins; among equal
// costs a free column (row4col == -1) beats an assigned one, the free one at the LARGEST position of `remaining` and the
// assigned one at the SMALLEST -- what the sequential scan `spc < lowest || (spc == lowest && row4col == -1)` keeps.
// rank encodes that preference (larger is better), -1 = no candidate.
constexpr int LSAP_FREE = 1 << 20;
__device__ __forceinline__ int lsap_rank(bool is_free, int it) { return is_free ? LSAP_FREE + it : LSAP_FREE - 1 - it; }
__device__ __forceinline__ int lsap_pos(int rank) { return rank >= LSAP_FREE ? rank - LSAP_FREE : LSAP_FREE - 1 - rank; }

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

// Gated cost of (detection i, track j) as the host Tracker builds it (tracker.py _gated_cost + hungarian_assignment):
// the greedy path's fp32 squared distance, widened to fp64, plus 1e18 when blocked, clamped to exactly 1e18 so that
// every blocked cell weighs the same.  Recomputed on every read: the T x K matrix is never stored.
__device__ __forceinline__ double gated_cost(const float* s_old, const float* s_px, const float* s_py, const float* s_isz,
                                             const float* s_tsz, const float* s_det, int i, int j) {
  const float* t = s_old + (size_t)j * TF;
  const float dx = __fsub_rn(t[CT_TRK_CT], s_px[i]), dy = __fsub_rn(t[CT_TRK_CT + 1], s_py[i]);
  const float dist = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
  const bool blocked = dist > s_tsz[j] || dist > s_isz[i] || t[CT_TRK_CLASS] != s_det[(size_t)i * TF + CT_TRK_CLASS];
  const double c = __dadd_rn((double)dist, blocked ? 1e18 : 0.0);
  return c > 1e18 ? 1e18 : c;
}

// --hungarian (tracker.py:52-72): the minimum-cost assignment of scipy.optimize.linear_sum_assignment, restated from
// Crouse's shortest augmenting path algorithm (IEEE TAES 52(4), 2016) with the same choice among equal-cost optima:
// rows = the smaller side (detections unless N > M), augmented in order, one Dijkstra search per row over the columns
// in `remaining` (initialised in reverse, swap-removed), fp64 reduced costs ((minVal + c) - u) - v.  Run by ONE warp:
// each search step is a shuffle min-reduction with the key of lsap_rank; the steps themselves are serial.
// Results: s_match[det] = track of a kept pair (cost <= 1e16), s_rej[det] = track of a rejected pair, s_taken[track]
// for both; the pairs are in ascending detection order, which is the order rejected tracks later coast in.
__device__ void hungarian_assign(const float* s_old, const float* s_px, const float* s_py, const float* s_isz,
                                 const float* s_tsz, const float* s_det, int N, int M, double* s_u, double* s_v,
                                 double* s_spc, int* s_path, int* s_c4r, int* s_r4c, int* s_rem, int* s_match,
                                 int* s_taken, int* s_rej, int* steps_out, int lane) {
  const bool tr = N > M;                                  // rows are the smaller side
  const int nr = tr ? M : N, nc = tr ? N : M;
  for (int j = lane; j < nc; j += 32) { s_v[j] = 0.0; s_r4c[j] = -1; }
  for (int i = lane; i < nr; i += 32) { s_u[i] = 0.0; s_c4r[i] = -1; }
  __syncwarp();
  int steps = 0;
  for (int cur = 0; cur < nr; ++cur) {
    for (int it = lane; it < nc; it += 32) { s_rem[it] = nc - 1 - it; s_spc[it] = CUDART_INF; }
    __syncwarp();
    double minVal = 0.0;
    int i = cur, sink = -1, nrem = nc;
    while (sink < 0) {                                    // terminates: a free column is always among `remaining`
      ++steps;
      const double ui = s_u[i];
      double best = CUDART_INF;
      int brank = -1;
      for (int it = lane; it < nrem; it += 32) {
        const int j = s_rem[it];
        const double c = tr ? gated_cost(s_old, s_px, s_py, s_isz, s_tsz, s_det, j, i)
                            : gated_cost(s_old, s_px, s_py, s_isz, s_tsz, s_det, i, j);
        const double r = __dsub_rn(__dsub_rn(__dadd_rn(minVal, c), ui), s_v[j]);
        double sp = s_spc[j];
        if (r < sp) { sp = r; s_spc[j] = r; s_path[j] = i; }
        const int rk = lsap_rank(s_r4c[j] < 0, it);
        if (sp < best || (sp == best && rk > brank)) { best = sp; brank = rk; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int orank = __shfl_xor_sync(0xffffffffu, brank, o);
        if (ov < best || (ov == best && orank > brank)) { best = ov; brank = orank; }
      }
      const int pos = lsap_pos(brank);
      const int j = s_rem[pos];
      minVal = best;
      const int owner = s_r4c[j];
      if (owner < 0) sink = j; else i = owner;
      --nrem;
      __syncwarp();
      if (lane == 0) { s_rem[pos] = s_rem[nrem]; s_rem[nrem] = j; }   // reached columns collect at the tail
      __syncwarp();
    }
    // duals: u[cur] += minVal; every other reached row (the owner of a reached column) and every reached column by
    // minVal - spc[column]
    for (int k = nrem + lane; k < nc; k += 32) {
      const int j = s_rem[k];
      const double dl = __dsub_rn(minVal, s_spc[j]);
      if (j != sink) s_u[s_r4c[j]] = __dadd_rn(s_u[s_r4c[j]], dl);
      s_v[j] = __dsub_rn(s_v[j], dl);
    }
    if (lane == 0) s_u[cur] = __dadd_rn(s_u[cur], minVal);
    __syncwarp();
    if (lane == 0) {                                      // augment back along the path
      int j = sink;
      for (;;) {
        const int r = s_path[j];
        s_r4c[j] = r;
        const int prev = s_c4r[r];
        s_c4r[r] = j;
        j = prev;
        if (r == cur) break;
      }
    }
    __syncwarp();
  }
  // pairs (det, track); > 1e16 means forced through a blocked cell: rejected
  for (int r = lane; r < nr; r += 32) {
    const int det = tr ? s_c4r[r] : r, trk = tr ? r : s_c4r[r];
    s_taken[trk] = 1;
    if (gated_cost(s_old, s_px, s_py, s_isz, s_tsz, s_det, det, trk) > 1e16) s_rej[det] = trk;
    else s_match[det] = trk;
  }
  if (steps_out && lane == 0) *steps_out = steps;
}

// --public_det births (tracker.py:83-103): public detection p = 0..P-1 claims argmin_i dist(pred_i, pub_p) over the
// unmatched, unclaimed detections (others read as (float)1e18; ties -> lowest i) when that distance is below the
// detection's box area.  Claimed detections get s_match = -2 and are listed in s_claim in claim order; returns their
// number.  One warp: the public centres are read 32 at a time and broadcast by shuffles.
__device__ int public_claims(const float* pc, int P, const float* s_px, const float* s_py, const float* s_isz, int N,
                             int* s_match, int* s_claim, int lane) {
  int n = 0;
  for (int base = 0; base < P && N > 0; base += 32) {
    float mx = 0.f, my = 0.f;
    if (base + lane < P) { mx = pc[2 * (base + lane)]; my = pc[2 * (base + lane) + 1]; }
    const int cnt = P - base < 32 ? P - base : 32;
    for (int q = 0; q < cnt; ++q) {
      const float qx = __shfl_sync(0xffffffffu, mx, q), qy = __shfl_sync(0xffffffffu, my, q);
      float best = CUDART_INF_F;
      int bi = 0x7fffffff;
      for (int i = lane; i < N; i += 32) {
        float v = 1e18f;
        if (s_match[i] == -1) {
          const float dx = __fsub_rn(s_px[i], qx), dy = __fsub_rn(s_py[i], qy);
          v = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
        }
        if (v < best) { best = v; bi = i; }               // ascending i per lane: first minimum kept
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov < best || (ov == best && oi < bi)) { best = ov; bi = oi; }
      }
      // a blocked argmin (only when every candidate is blocked) is never claimed
      const bool claim = bi < N && best < s_isz[bi] && s_match[bi] == -1;
      __syncwarp();
      if (claim && lane == 0) { s_match[bi] = -2; s_claim[n] = bi; }
      n += claim ? 1 : 0;
      __syncwarp();
    }
  }
  return n;
}

// The payload row of one detection (ct_track_payload's field order), generic_post_process's fp32 arithmetic
// (post_process.py:55-89, ddd_utils.py:91-136): r = its record, ct = its (amodal) image centre, P = the stream's calib.
__device__ __forceinline__ void det_payload(const ct_track_payload& p, const float* r, const float* to,
                                            const float* ct, const float* P, float* out) {
  int o = 0;
  if (p.rec_hps >= 0)
    for (int k = 0; k < p.hps_floats; k += 2) {
      const float x = r[p.rec_hps + k], y = r[p.rec_hps + k + 1];
      out[o++] = aff_f32(to, x, y);
      out[o++] = aff_f32(to + 3, x, y);
    }
  if (p.rec_dep >= 0) out[o++] = r[p.rec_dep];
  if (p.rec_dim >= 0)
    for (int k = 0; k < 3; ++k) out[o++] = r[p.rec_dim + k];
  float alpha = 0.f;
  // np.arctan2 on float32 operands is atan2f here (within 3 ulp; an fp64 atan2 put the kernel on a stack frame)
  if (p.rec_rot >= 0) {          // get_alpha: bin 1 when rot[1] > rot[5]; the +-pi/2 is a float32 constant
    const float* q = r + p.rec_rot;
    const float hp = (float)(0.5 * CUDART_PI);
    alpha = q[1] > q[5] ? __fadd_rn(atan2f(q[2], q[3]), -hp) : __fadd_rn(atan2f(q[6], q[7]), hp);
    out[o++] = alpha;
  }
  if (p.rec_rot >= 0 && p.rec_dep >= 0 && p.rec_dim >= 0) {
    // ddd2locrot: unproject_2d_to_3d in fp32, loc[1] += dim[0] / 2, then alpha2rot_y (alpha is fp64 there)
    const float dep = r[p.rec_dep];
    const float z = __fsub_rn(dep, P[11]);
    const float x = __fdiv_rn(__fsub_rn(__fsub_rn(__fmul_rn(ct[0], dep), P[3]), __fmul_rn(P[2], z)), P[0]);
    const float y = __fdiv_rn(__fsub_rn(__fsub_rn(__fmul_rn(ct[1], dep), P[7]), __fmul_rn(P[6], z)), P[5]);
    out[o++] = x;
    out[o++] = __fadd_rn(y, __fmul_rn(r[p.rec_dim], 0.5f));
    out[o++] = z;
    double ry = (double)alpha + (double)atan2f(__fsub_rn(ct[0], P[2]), P[0]);
    if (ry > CUDART_PI) ry -= 2 * CUDART_PI;
    if (ry < -CUDART_PI) ry += 2 * CUDART_PI;
    out[o++] = (float)ry;
  }
  if (p.rec_velocity >= 0)
    for (int k = 0; k < p.velocity_floats; ++k) out[o++] = r[p.rec_velocity + k];
  if (p.rec_nuscenes_att >= 0)
    for (int k = 0; k < p.att_floats; ++k) out[o++] = r[p.rec_nuscenes_att + k];
}

// Boxes of the NEXT frame's prior heat-map (detector.py:254-290) from stream b's first `total` track rows `trk`: image
// -> input coords, clip, radius, centre; rows past `total` and tracks that are not splatted get radius -1.  The one copy
// of this arithmetic: the track step and ct_track_start both end with it.  Called by all TRK_THREADS threads.
__device__ __forceinline__ void track_boxes(const ct_track_desc& d, int b, const float* trk, int total, int tid) {
  if (!d.boxes) return;
  const int T = d.max_tracks;
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

// PAY: also write the payload table (ct_track_step_payload); the 2-D head sets run the <false> instantiation.
template <bool PAY>
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
  // association scratch, present only when ct_track_step_assoc enables a mode (ct_track_assoc_smem_bytes)
  double* s_u = reinterpret_cast<double*>(tsm + trk_base_bytes(K, T));   // [K] row duals
  double* s_v = s_u + K;                                        // [T] column duals
  double* s_spc = s_v + T;                                      // [T] shortest-path costs of the current search
  int* s_path = reinterpret_cast<int*>(s_spc + T);              // [T] predecessor row of a column
  int* s_c4r = s_path + T;                                      // [K] column of a row or -1
  int* s_r4c = s_c4r + K;                                       // [T] row of a column or -1
  int* s_rem = s_r4c + T;                                       // [T] columns not yet reached, then the reached ones
  int* s_rej = s_rem + T;                                       // [K] track of a det's rejected Hungarian pair or -1
  int* s_claim = s_rej + K;                                     // [K] detections claimed by public detections, in order
  __shared__ float red_v[TRK_THREADS / 32];
  __shared__ int red_j[TRK_THREADS / 32];
  __shared__ int s_n, s_total, s_ids, s_nclaim;

  int M = d.counts[b * 2 + 0];
  if (M > T) M = T;
  const int id_count = d.counts[b * 2 + 1];
  float* trk = d.tracks + (size_t)b * T * TF;
  for (int i = tid; i < M * TF; i += TRK_THREADS) s_old[i] = trk[i];
  // payload rows are permuted in place like the track rows: the old ones are staged before any is written
  const int Wp = PAY ? a.p.width : 0;
  float* pay = PAY ? a.p.payload + (size_t)b * T * Wp : nullptr;
  float* s_oldp = reinterpret_cast<float*>(tsm + a.pay_smem);  // [T][Wp]
  if constexpr (PAY)
    for (int i = tid; i < M * Wp; i += TRK_THREADS) s_oldp[i] = pay[i];
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
  const bool amodal = PAY && a.p.rec_rot >= 0 && a.p.rec_dep >= 0 && a.p.rec_dim >= 0;
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
    float acx = ctx, acy = cty;
    if (amodal) {      // post_process.py:76-84: ct becomes the amodal centre after `tracking` was taken from the peak
      if (a.p.rec_amodel_offset >= 0) {   // numpy's fp32 mean of the two output-grid corners + amodel_offset
        const float mx = __fadd_rn(__fmul_rn(__fadd_rn(bl, br), 0.5f), r[a.p.rec_amodel_offset]);
        const float my = __fadd_rn(__fmul_rn(__fadd_rn(bt, bb), 0.5f), r[a.p.rec_amodel_offset + 1]);
        acx = aff_f32(to, mx, my); acy = aff_f32(to + 3, mx, my);
      } else {                            // the image box centre
        acx = __fmul_rn(__fadd_rn(o[CT_TRK_BBOX], o[CT_TRK_BBOX + 2]), 0.5f);
        acy = __fmul_rn(__fadd_rn(o[CT_TRK_BBOX + 1], o[CT_TRK_BBOX + 3]), 0.5f);
      }
      o[CT_TRK_CT] = acx; o[CT_TRK_CT + 1] = acy;
    }
    s_px[i] = __fadd_rn(acx, tx);
    s_py[i] = __fadd_rn(acy, ty);
    s_isz[i] = __fmul_rn(__fsub_rn(o[CT_TRK_BBOX + 2], o[CT_TRK_BBOX]), __fsub_rn(o[CT_TRK_BBOX + 3], o[CT_TRK_BBOX + 1]));
    s_match[i] = -1;
  }
  for (int j = tid; j < M; j += TRK_THREADS) {
    const float* t = s_old + (size_t)j * TF;
    s_tsz[j] = __fmul_rn(__fsub_rn(t[CT_TRK_BBOX + 2], t[CT_TRK_BBOX]), __fsub_rn(t[CT_TRK_BBOX + 3], t[CT_TRK_BBOX + 1]));
    s_taken[j] = 0;
  }
  __syncthreads();

  const bool hung = a.as.hungarian != 0, pub = a.as.public_det != 0;
  if (hung || pub) {
    for (int i = tid; i < N; i += TRK_THREADS) s_rej[i] = -1;
    __syncthreads();
  }
  if (!hung && tid == 0 && a.as.steps) a.as.steps[b] = 0;
  const float INF = 3.0e38f;
  if (hung) {
    if (warp == 0) hungarian_assign(s_old, s_px, s_py, s_isz, s_tsz, s_det, N, M, s_u, s_v, s_spc, s_path, s_c4r, s_r4c,
                                    s_rem, s_match, s_taken, s_rej, a.as.steps ? a.as.steps + b : nullptr, lane);
    __syncthreads();
  }
  // ---- greedy assignment (tracker.py:129-138): detections in score order take their nearest free, valid track;
  //      argmin ties -> lowest track index
  for (int i = 0; i < N && M > 0 && !hung; ++i) {
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

  // ---- MOT public-detection births (tracker.py:83-103): each public detection, in order, claims its nearest
  //      unmatched detection if closer than that detection's box area
  if (pub) {
    if (warp == 0) {
      int P = a.as.public_n[b];
      P = P < 0 ? 0 : (P > a.as.max_public ? a.as.max_public : P);
      const int n = public_claims(a.as.public_ct + (size_t)b * a.as.max_public * 2, P, s_px, s_py, s_isz, N, s_match,
                                  s_claim, lane);
      if (lane == 0) s_nclaim = n;
    }
    __syncthreads();
  }

  // ---- output order (tracker.py:74-127): matched detections, then new tracks, then coasting tracks.  Births and
  //      coasting walk the reference's `unmatched` lists: the naturally unmatched ascending, then the detections /
  //      tracks of rejected (forced through a blocked cell) Hungarian pairs in pair order
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
    auto birth = [&](int i) {
      float* o = s_det + (size_t)i * TF;
      if (o[CT_TRK_SCORE] > d.new_thresh) {
        ++ids;
        o[CT_TRK_ID] = (float)ids; o[CT_TRK_AGE] = 1.f; o[CT_TRK_ACTIVE] = 1.f;
        if (pos < T) s_pos_det[i] = pos++;
      }
    };
    auto coast = [&](int j) {
      float* t = s_old + (size_t)j * TF;
      if (t[CT_TRK_AGE] < (float)d.max_age) {
        t[CT_TRK_AGE] += 1.f; t[CT_TRK_ACTIVE] = 0.f;
        if (pos < T) s_pos_trk[j] = pos++;
      }
    };
    if (pub) {
      for (int k = 0; k < s_nclaim; ++k) birth(s_claim[k]);
    } else {
      for (int i = 0; i < N; ++i)
        if (s_match[i] < 0 && !(hung && s_rej[i] >= 0)) birth(i);
      if (hung)
        for (int i = 0; i < N; ++i)
          if (s_rej[i] >= 0) birth(i);
    }
    for (int j = 0; j < M; ++j) {
      s_pos_trk[j] = -1;
      if (!s_taken[j]) coast(j);
    }
    if (hung)
      for (int i = 0; i < N; ++i)
        if (s_rej[i] >= 0) coast(s_rej[i]);
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
  if constexpr (PAY) {           // detections: computed from the read-only records; coasting tracks: their staged rows
    const float* P = a.p.calib ? a.p.calib + b * 12 : nullptr;
    for (int i = tid; i < N; i += TRK_THREADS)
      if (s_pos_det[i] >= 0)
        det_payload(a.p, rec + (size_t)i * d.F, to, s_det + (size_t)i * TF + CT_TRK_CT, P, pay + (size_t)s_pos_det[i] * Wp);
    for (int e = tid; e < M * Wp; e += TRK_THREADS) {
      const int j = e / Wp, f = e - j * Wp;
      if (s_pos_trk[j] >= 0) pay[(size_t)s_pos_trk[j] * Wp + f] = s_oldp[e];
    }
  }
  if (tid == 0) { d.counts[b * 2 + 0] = total; d.counts[b * 2 + 1] = s_ids; }
  __syncthreads();     // the table rows written above are re-read below by other threads
  __threadfence_block();
  track_boxes(d, b, trk, total, tid);
}

// ct_track_start: stream starts[e][0] begins a new video -- Tracker.reset + init_track(seeds): its T track rows, counts
// and payload rows are cleared, its starts[e][1] seed rows (already filtered and numbered on the host) written, and its
// render boxes computed from them by the same code as the track step's.  One CTA per started stream; the seeds of
// entry e follow those of entries 0..e-1 in `seeds`.
__global__ void __launch_bounds__(TRK_THREADS)
track_start_kernel(const ct_track_desc d, float* __restrict__ payload, int Wp, const int* __restrict__ starts,
                   const float* __restrict__ seeds) {
  const int e = blockIdx.x, tid = threadIdx.x, T = d.max_tracks;
  const int b = starts[2 * e];
  if (b < 0 || b >= d.B) return;
  auto clamp_n = [&](int n) { return seeds == nullptr ? 0 : (n < 0 ? 0 : (n > T ? T : n)); };
  size_t off = 0;
  for (int k = 0; k < e; ++k) off += (size_t)clamp_n(starts[2 * k + 1]);
  const int n = clamp_n(starts[2 * e + 1]);
  float* trk = d.tracks + (size_t)b * T * TF;
  const float* src = seeds ? seeds + off * TF : nullptr;
  for (int i = tid; i < T * TF; i += TRK_THREADS) trk[i] = i < n * TF ? src[i] : 0.f;
  if (payload)
    for (int i = tid; i < T * Wp; i += TRK_THREADS) payload[(size_t)b * T * Wp + i] = 0.f;
  if (tid == 0) { d.counts[b * 2 + 0] = n; d.counts[b * 2 + 1] = n; }
  __syncthreads();     // the seed rows written above are re-read below by other threads
  __threadfence_block();
  track_boxes(d, b, trk, n, tid);
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

// The warped uint8 BGR value of output pixel (x, y): src uint8 [sh, sw, 3] with row pitch sstep bytes, M the inverted
// (dst -> src) map.  The one copy of the per-pixel warp arithmetic: ct_warp_affine_normalize and ct_pack_stem_frames
// both call it, so that the fused stem input is byte-identical to the fp32 image packed afterwards.
__device__ __forceinline__ void warp_bilinear_u8(const unsigned char* __restrict__ img, int sh, int sw, int sstep,
                                                 const double* M, int x, int y, int p8[3]) {
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
    p8[c] = pix < 0 ? 0 : (pix > 255 ? 255 : pix);
  }
}

// ((inp / 255. - mean) / std).astype(float32): float64 arithmetic, one final rounding
__device__ __forceinline__ float normalize_u8(int v, float mean, float stdv) {
  return (float)(((double)v / 255.0 - (double)mean) / (double)stdv);
}

__global__ void warp_affine_norm_kernel(const unsigned char* __restrict__ src, int sh, int sw, int sstep,
                                        float* __restrict__ dst, int B, int oh, int ow,
                                        const double* __restrict__ minv /*[B][6] dst->src*/, float3 mean, float3 stdv) {
  const size_t total = (size_t)B * oh * ow;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / ((size_t)oh * ow));
    const size_t r = i - (size_t)b * oh * ow;
    const int y = (int)(r / ow), x = (int)(r - (size_t)y * ow);
    int p8[3];
    warp_bilinear_u8(src + (size_t)b * sh * sstep, sh, sw, sstep, minv + b * 6, x, y, p8);
    const size_t plane = (size_t)oh * ow;
    float* o = dst + (size_t)b * 3 * plane + (size_t)y * ow + x;
    o[0] = normalize_u8(p8[0], mean.x, stdv.x);
    o[plane] = normalize_u8(p8[1], mean.y, stdv.y);
    o[2 * plane] = normalize_u8(p8[2], mean.z, stdv.z);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// ct_pack_stem_frames: the tensor-core stem's input [B,H,W,8] bf16 = (norm(warp(cur_b)) x3, norm(warp(prev_b)) x3,
// pre_hm, 0) straight from each stream's uint8 frame.  blockIdx.y = stream (its descriptor read once, from the kernel
// parameters), one 16-byte output pixel per thread and iteration.  The normalisation depends on the 8-bit value only:
// a 3 x 256 table built per CTA with normalize_u8 gives the same floats without a per-pixel fp64 divide.
// FLIP (ct_pack_stem_frames_flip): out is [2B,H,W,8] and image B+b is image b mirrored.  The mirrored packed pixel
// (y, W-1-x) equals the original's (y, x) in all 8 channels (frame, previous frame and pre_hm are all mirrored), so each
// pixel is warped once and its 16-byte vector stored twice.
// ------------------------------------------------------------------------------------------------------------------
struct FramesArgs {
  ct_frame f[CT_FRAMES_PER_LAUNCH];
};

constexpr int PACK_THREADS = 256;
constexpr int PACK_PIX_PER_THREAD = 4;      // pixels per thread: amortises the table build over 1024 pixels per CTA

template <bool FLIP>
__global__ void __launch_bounds__(PACK_THREADS)
pack_stem_frames_kernel(const unsigned char* __restrict__ cur, const unsigned char* __restrict__ prev,
                        const __grid_constant__ FramesArgs fa, int b0, int B, float3 mean, float3 stdv,
                        const float* __restrict__ hm, uint4* __restrict__ out, int H, int W) {
  __shared__ float tab[3][256];
  for (int i = threadIdx.x; i < 3 * 256; i += PACK_THREADS) {
    const int c = i >> 8, v = i & 255;
    tab[c][v] = normalize_u8(v, c == 0 ? mean.x : (c == 1 ? mean.y : mean.z), c == 0 ? stdv.x : (c == 1 ? stdv.y : stdv.z));
  }
  __syncthreads();
  const ct_frame& f = fa.f[blockIdx.y];
  const int b = b0 + blockIdx.y;
  const size_t plane = (size_t)H * W;
  const unsigned char* src = cur + f.offset;
  const unsigned char* psrc = prev ? prev + f.offset : nullptr;
  const size_t base = (size_t)blockIdx.x * PACK_THREADS * PACK_PIX_PER_THREAD + threadIdx.x;
#pragma unroll
  for (int k = 0; k < PACK_PIX_PER_THREAD; ++k) {
    const size_t r = base + (size_t)k * PACK_THREADS;
    if (r >= plane) break;
    const int y = (int)(r / W), x = (int)(r - (size_t)y * W);
    float v[8];
    int p8[3];
    warp_bilinear_u8(src, f.h, f.w, f.step, f.minv, x, y, p8);
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = tab[c][p8[c]];
    if (psrc) {
      warp_bilinear_u8(psrc, f.h, f.w, f.step, f.minv, x, y, p8);
#pragma unroll
      for (int c = 0; c < 3; ++c) v[3 + c] = tab[c][p8[c]];
    } else {
      v[3] = v[4] = v[5] = 0.f;
    }
    v[6] = hm ? __ldg(hm + (size_t)b * plane + r) : 0.f;
    v[7] = 0.f;
    uint4 o;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
    for (int q = 0; q < 4; ++q) h[q] = __floats2bfloat162_rn(v[2 * q], v[2 * q + 1]);
    out[(size_t)b * plane + r] = o;
    if constexpr (FLIP) out[(size_t)(B + b) * plane + (size_t)y * W + (W - 1 - x)] = o;
  }
}

}  // namespace ctb

using namespace ctb;

static inline int sw_blocks(size_t total) {
  size_t b = (total + 255) / 256;
  const size_t cap = (size_t)device_sm_count() * 16;
  return (int)(b < cap ? (b ? b : 1) : cap);
}

extern "C" int ct_flip_merge_heads(const ct_flip_head* heads, int32_t n_heads, int32_t B, int32_t H, int32_t W,
                                   void* stream) {
  CT_REQUIRE(heads, "null pointer");
  CT_REQUIRE(n_heads > 0 && n_heads <= CT_FLIP_MAX_HEADS, "n_heads outside [1, CT_FLIP_MAX_HEADS]");
  CT_REQUIRE(B > 0 && H > 0 && W > 0, "bad shape");
  FlipArgs fa = {};
  size_t most = 0;
  for (int32_t i = 0; i < n_heads; ++i) {
    CT_REQUIRE(heads[i].in && heads[i].out, "null pointer");
    CT_REQUIRE(heads[i].C > 0, "bad shape");
    fa.h[i] = heads[i];
    const size_t n = (size_t)B * heads[i].C * H * W;
    most = n > most ? n : most;
  }
  dim3 grid((unsigned)sw_blocks(most), (unsigned)n_heads);
  flip_merge_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(fa, B, H, W);
  return after_launch();
}

extern "C" int ct_flip_merge(const float* in2, float* out, int32_t C, int32_t H, int32_t W, const int32_t* perm,
                             const float* sign, void* stream) {
  const ct_flip_head h = {in2, out, C, 0, perm, sign};
  return ct_flip_merge_heads(&h, 1, 1, H, W, stream);
}

extern "C" int ct_mirror_x(const float* src, float* dst, int32_t n, int32_t C, int32_t H, int32_t W, void* stream) {
  CT_REQUIRE(src && dst, "null pointer");
  CT_REQUIRE(n > 0 && C > 0 && H > 0 && W > 0, "bad shape");
  const size_t rows = (size_t)n * C * H;
  mirror_x_kernel<<<sw_blocks(rows * W), 256, 0, (cudaStream_t)stream>>>(src, dst, rows, W);
  return after_launch();
}

extern "C" int64_t ct_track_smem_bytes(int32_t K, int32_t max_tracks) {
  return (int64_t)((size_t)max_tracks * TF + (size_t)K * TF + 3 * (size_t)K + max_tracks) * 4 +
         (int64_t)(2 * (size_t)K + 2 * (size_t)max_tracks) * 4 + 64;
}

extern "C" int64_t ct_track_assoc_smem_bytes(int32_t K, int32_t max_tracks) {
  return ct_track_smem_bytes(K, max_tracks) + (int64_t)(8 * ((size_t)K + 2 * (size_t)max_tracks)) +
         (int64_t)(4 * (3 * (size_t)max_tracks + 3 * (size_t)K));
}

extern "C" int64_t ct_track_payload_smem_bytes(int32_t K, int32_t max_tracks, int32_t width, int32_t assoc) {
  return (assoc ? ct_track_assoc_smem_bytes(K, max_tracks) : ct_track_smem_bytes(K, max_tracks)) +
         (int64_t)max_tracks * width * 4;
}

// a record field of `w` floats at `off` (-1 = absent) lies inside the heads part of an F-float record
static inline bool rec_field_ok(int32_t off, int32_t w, int32_t F) {
  return off < 0 || (w > 0 && off >= CT_REC_HEADS && off + w <= F);
}

extern "C" int ct_track_step_payload(const ct_track_desc* d, const ct_track_assoc* as, const ct_track_payload* p,
                                     void* stream) {
  CT_REQUIRE(d && as && d->records && d->trans_out_inv && d->tracks && d->counts, "null pointer");
  CT_REQUIRE(d->B > 0 && d->K > 0 && d->F >= CT_REC_HEADS && d->max_tracks >= d->K, "bad shape");
  CT_REQUIRE(d->rec_tracking < 0 || d->rec_tracking + 2 <= d->F, "tracking offset outside the record");
  CT_REQUIRE(d->boxes == nullptr || (d->trans_input != nullptr && d->inp_h > 0 && d->inp_w > 0), "boxes need trans_input");
  CT_REQUIRE(!as->public_det || (as->public_ct && as->public_n), "public_det needs public_ct and public_n");
  CT_REQUIRE(!as->public_det || as->max_public > 0, "public_det needs max_public > 0");
  if (p) {
    CT_REQUIRE(p->payload, "null payload table");
    CT_REQUIRE(rec_field_ok(p->rec_hps, p->hps_floats, d->F) && (p->rec_hps < 0 || p->hps_floats % 2 == 0) &&
               rec_field_ok(p->rec_dep, 1, d->F) && rec_field_ok(p->rec_dim, 3, d->F) &&
               rec_field_ok(p->rec_rot, 8, d->F) && rec_field_ok(p->rec_amodel_offset, 2, d->F) &&
               rec_field_ok(p->rec_velocity, p->velocity_floats, d->F) &&
               rec_field_ok(p->rec_nuscenes_att, p->att_floats, d->F), "payload field outside the record");
    const bool ddd = p->rec_rot >= 0 && p->rec_dep >= 0 && p->rec_dim >= 0;
    const int64_t w = (p->rec_hps >= 0 ? p->hps_floats : 0) + (p->rec_dep >= 0 ? 1 : 0) + (p->rec_dim >= 0 ? 3 : 0) +
                      (p->rec_rot >= 0 ? 1 : 0) + (ddd ? 4 : 0) + (p->rec_velocity >= 0 ? p->velocity_floats : 0) +
                      (p->rec_nuscenes_att >= 0 ? p->att_floats : 0);
    CT_REQUIRE(w > 0 && p->width == w, "payload width does not match its fields");
    CT_REQUIRE(!ddd || p->calib, "rot, dep and dim need calib");
  }
  const bool scratch = as->hungarian || as->public_det;
  const size_t smem = (size_t)ct_track_payload_smem_bytes(d->K, d->max_tracks, p ? p->width : 0, scratch);
  CT_REQUIRE(smem <= 200 * 1024, "track table does not fit in shared memory (lower max_tracks)");
  auto kernel = p ? track_step_kernel<true> : track_step_kernel<false>;
  if (smem > 48 * 1024)
    CT_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  TrackArgs a = {};
  a.d = *d;
  a.as = *as;
  if (p) a.p = *p;
  a.pay_smem = (int)(trk_base_bytes(d->K, d->max_tracks) +
                     (scratch ? ct_track_assoc_smem_bytes(d->K, d->max_tracks) - ct_track_smem_bytes(d->K, d->max_tracks)
                              : 0));
  kernel<<<d->B, TRK_THREADS, smem, (cudaStream_t)stream>>>(a);
  return after_launch();
}

extern "C" int ct_track_step_assoc(const ct_track_desc* d, const ct_track_assoc* as, void* stream) {
  return ct_track_step_payload(d, as, nullptr, stream);
}

extern "C" int ct_track_step(const ct_track_desc* d, void* stream) {
  const ct_track_assoc greedy = {};
  return ct_track_step_assoc(d, &greedy, stream);
}

extern "C" int ct_track_start(const ct_track_desc* d, const ct_track_payload* p, const int32_t* starts,
                              int32_t n_starts, const float* seeds, void* stream) {
  CT_REQUIRE(d && d->tracks && d->counts, "null pointer");
  CT_REQUIRE(d->B > 0 && d->max_tracks > 0, "bad shape");
  CT_REQUIRE(d->boxes == nullptr || (d->trans_input != nullptr && d->inp_h > 0 && d->inp_w > 0), "boxes need trans_input");
  CT_REQUIRE(n_starts >= 0 && n_starts <= d->B, "n_starts outside [0, B]");
  CT_REQUIRE(n_starts == 0 || starts, "null start list");
  CT_REQUIRE(!p || (p->payload && p->width > 0), "payload table needs payload and width > 0");
  if (n_starts == 0) return CT_OK;
  track_start_kernel<<<n_starts, TRK_THREADS, 0, (cudaStream_t)stream>>>(*d, p ? p->payload : nullptr, p ? p->width : 0,
                                                                          starts, seeds);
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

template <bool FLIP>
static int pack_stem_frames(const uint8_t* cur, const uint8_t* prev, const ct_frame* frames, int32_t B,
                            const float* mean, const float* std, const float* pre_hm, void* out, int32_t H, int32_t W,
                            void* stream) {
  CT_REQUIRE(cur && frames && mean && std && out, "null pointer");
  CT_REQUIRE(B > 0 && H > 0 && W > 0, "bad shape");
  for (int32_t b = 0; b < B; ++b)
    CT_REQUIRE(frames[b].offset >= 0 && frames[b].h > 0 && frames[b].w > 0 && frames[b].step >= 3 * frames[b].w,
               "bad frame descriptor (offset >= 0, h > 0, w > 0, step >= 3 w)");
  const size_t plane = (size_t)H * W;
  const size_t per_cta = (size_t)PACK_THREADS * PACK_PIX_PER_THREAD;
  CT_REQUIRE((plane + per_cta - 1) / per_cta <= 0x7fffffffu, "output too large");
  const float3 m = make_float3(mean[0], mean[1], mean[2]), s = make_float3(std[0], std[1], std[2]);
  // descriptors travel in the kernel parameters (captured by value in a CUDA graph): CT_FRAMES_PER_LAUNCH per launch
  for (int32_t b0 = 0; b0 < B; b0 += CT_FRAMES_PER_LAUNCH) {
    const int n = B - b0 < CT_FRAMES_PER_LAUNCH ? B - b0 : CT_FRAMES_PER_LAUNCH;
    FramesArgs fa = {};
    memcpy(fa.f, frames + b0, sizeof(ct_frame) * n);
    dim3 grid((unsigned)((plane + per_cta - 1) / per_cta), (unsigned)n);
    pack_stem_frames_kernel<FLIP><<<grid, PACK_THREADS, 0, (cudaStream_t)stream>>>(cur, prev, fa, b0, B, m, s, pre_hm,
                                                                                   (uint4*)out, H, W);
    const int rc = after_launch();
    if (rc != CT_OK) return rc;
  }
  return CT_OK;
}

extern "C" int ct_pack_stem_frames(const uint8_t* cur, const uint8_t* prev, const ct_frame* frames, int32_t B,
                                   const float* mean, const float* std, const float* pre_hm, void* out, int32_t H,
                                   int32_t W, void* stream) {
  return pack_stem_frames<false>(cur, prev, frames, B, mean, std, pre_hm, out, H, W, stream);
}

extern "C" int ct_pack_stem_frames_flip(const uint8_t* cur, const uint8_t* prev, const ct_frame* frames, int32_t B,
                                        const float* mean, const float* std, const float* pre_hm, void* out, int32_t H,
                                        int32_t W, void* stream) {
  return pack_stem_frames<true>(cur, prev, frames, B, mean, std, pre_hm, out, H, W, stream);
}
