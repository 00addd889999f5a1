// Per-stream state kept on the device between frames (SURVEY 8f rows 1-3):
//   ct_track_step    generic_post_process's affine + Tracker.step's greedy displacement association
//                    (utils/post_process.py:21-91, utils/tracker.py:28-138) on the packed decode records, plus the
//                    (centre, radius) boxes of Detector._get_additional_inputs (detector.py:254-290) for the NEXT frame;
//                    ct_track_step_assoc: the same kernel with --hungarian (scipy's linear_sum_assignment restated,
//                    one warp) and / or --public_det births (tracker.py:52-72,83-103); ct_track_step_payload: also
//                    the pose / 3D / velocity / attribute fields of generic_post_process (post_process.py:55-89) in a
//                    payload table beside the track table, and the amodal centre on 3D head sets
//   ct_render_tracks the gaussian max-splat of those boxes into pre_hm (image.py:128-154)
//   ct_track_start / ct_track_restore   a stream's table reset and seeded, or restored verbatim from an exported one
//   ct_track_step_mapped / ct_render_tracks_mapped   the same two on a compacted batch of live streams (image i =
//                    stream streams[i]), for StreamRunner's idle streams
//   ct_post_process  Detector.post_process + merge_outputs (detector.py:356-377) for runners without a tracker: the
//                    track step's per-detection affine and payload fields, each stream's kept records in parallel
//   ct_flip_merge    Detector._flip_output (detector.py:311-332; model/utils.py:28-50) for --flip_test;
//                    ct_flip_merge_heads: every averaged head of B (frame, mirror) pairs in one launch
//   ct_mirror_x      the mirrored half of a --flip_test batch (detector.py:225-226,285-286)
//   ct_warp_affine_normalize   Detector.pre_process's cv2.warpAffine(INTER_LINEAR) + (x/255 - mean)/std + HWC->CHW
//                    (detector.py:207-226), cv2's fixed-point bilinear restated
//   ct_pack_stem_frames_dev    the same warp + normalise of B ragged uint8 frames (and of their previous frames) that
//                    device-resident descriptors describe, written straight as the tensor-core stem's packed bf16
//                    input; ct_pack_stem_frames_flip_dev also writes each stream's mirror image (--flip_test);
//                    ct_warp_frames_normalize the same frames into an fp32 image.  BGR, NV12 or I420 frames, the
//                    latter two with cv2.cvtColor(COLOR_YUV2BGR_NV12 / _I420) applied to each bilinear tap
//   ct_stage_frames  B frames already in device memory (a GPU decoder's) copied into a frame slot in its layout
//   ct_crop_boxes    each stream's active tracks (or kept detections) cropped out of its frame slot: cv2.warpAffine
//                    of the box stretched to a fixed crop size, the frames kernels' bilinear taps;
//                    ct_crop_boxes_tensor the same crops as one packed, normalised fp32 / fp16 / bf16 NCHW batch
// All HBM-bound byte/index work: one pass over the data, coalesced, no tensor cores.
#include <cuda_fp16.h>
#include <math_constants.h>

#include <type_traits>

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
  const int* streams;      // ct_track_step_mapped: CTA i runs stream streams[i] on records[i]; NULL = identity
  int n_streams;           // rows of every per-stream array when streams != NULL
  const ct_track_opts* opts;   // ct_track_step_opts: stream b's settings are opts[b]; NULL = `dflt`
  ct_track_opts dflt;      // the descriptor's scalars and the assoc modes (the entry points without opts)
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

// generic_post_process (post_process.py:21-91) of one record r: the first CT_DET_FLOATS columns of its result row --
// score, class + 1, ct, tracking, bbox -- in image coordinates through the output affine `to`.  amodal (3D head sets,
// post_process.py:76-84): ct becomes the amodal centre after `tracking` was taken from the heat-map peak; the output-grid
// box centre + amodel_offset (rec_amodel_offset >= 0) or the image box centre.  (acx, acy) = the written ct, (tx, ty) =
// the written tracking, for the track step's association.  The one copy of this arithmetic: the track step and
// ct_post_process both call it.
__device__ __forceinline__ void det_row(const float* r, const float* to, int rec_tracking, bool amodal,
                                        int rec_amodel_offset, float* o, float& acx, float& acy, float& tx, float& ty) {
  const float cx = r[CT_REC_XS], cy = r[CT_REC_YS];
  const float ctx = aff_f32(to, cx, cy), cty = aff_f32(to + 3, cx, cy);
  tx = 0.f, ty = 0.f;
  if (rec_tracking >= 0) {
    const float px = __fadd_rn(r[rec_tracking], cx), py = __fadd_rn(r[rec_tracking + 1], cy);
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
  acx = ctx, acy = cty;
  if (amodal) {
    if (rec_amodel_offset >= 0) {         // numpy's fp32 mean of the two output-grid corners + amodel_offset
      const float mx = __fadd_rn(__fmul_rn(__fadd_rn(bl, br), 0.5f), r[rec_amodel_offset]);
      const float my = __fadd_rn(__fmul_rn(__fadd_rn(bt, bb), 0.5f), r[rec_amodel_offset + 1]);
      acx = aff_f32(to, mx, my); acy = aff_f32(to + 3, mx, my);
    } else {                              // the image box centre
      acx = __fmul_rn(__fadd_rn(o[CT_TRK_BBOX], o[CT_TRK_BBOX + 2]), 0.5f);
      acy = __fmul_rn(__fadd_rn(o[CT_TRK_BBOX + 1], o[CT_TRK_BBOX + 3]), 0.5f);
    }
    o[CT_TRK_CT] = acx; o[CT_TRK_CT + 1] = acy;
  }
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
__device__ __forceinline__ void track_boxes(const ct_track_desc& d, int b, const float* trk, int total, float pre_thresh,
                                            int tid) {
  if (!d.boxes) return;
  const int T = d.max_tracks;
  const double* ti = d.trans_input + b * 6;
  float* bx = d.boxes + (size_t)b * T * 5;
  for (int r = tid; r < T; r += TRK_THREADS) {
    float radius = -1.f, cxo = 0.f, cyo = 0.f;
    if (r < total) {
      const float* t = trk + (size_t)r * TF;
      if (!(t[CT_TRK_SCORE] < pre_thresh) && t[CT_TRK_ACTIVE] != 0.f) {
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
// MAP: ct_track_step_mapped (a.streams); a template parameter so that the identity instantiations stay as they were.
template <bool PAY, bool MAP = false>
__global__ void __launch_bounds__(TRK_THREADS)
track_step_kernel(const TrackArgs a) {
  extern __shared__ __align__(16) unsigned char tsm[];
  const ct_track_desc& d = a.d;
  // b indexes every per-stream array; the CTA's records are always records[blockIdx.x]
  const int b = MAP ? a.streams[blockIdx.x] : blockIdx.x;
  if (MAP && (b < 0 || b >= a.n_streams)) return;           // a padding image, or no stream: nothing is written
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
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
  // the stream's settings, read once per CTA and kept in shared memory (held in registers across the association they
  // pushed the payload instantiation into spills)
  __shared__ ct_track_opts so;

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
  if (tid == 0) {
    s_n = 0;
    so = a.opts ? a.opts[b] : a.dflt;
  }
  __syncthreads();

  // ---- detections of this frame: generic_post_process (post_process.py:21-91), merge_outputs (detector.py:371-377)
  const float* rec = d.records + (size_t)(MAP ? (int)blockIdx.x : b) * K * d.F;
  const float* to = d.trans_out_inv + b * 6;
  int cnt = 0;
  for (int i = tid; i < K; i += TRK_THREADS) cnt += rec[(size_t)i * d.F + CT_REC_SCORE] > so.out_thresh ? 1 : 0;
  atomicAdd(&s_n, cnt);
  __syncthreads();
  const int N = s_n;                     // records are sorted by score: the kept detections are a prefix
  const bool amodal = PAY && a.p.rec_rot >= 0 && a.p.rec_dep >= 0 && a.p.rec_dim >= 0;
  for (int i = tid; i < N; i += TRK_THREADS) {
    float* o = s_det + (size_t)i * TF;
    float acx, acy, tx, ty;
    det_row(rec + (size_t)i * d.F, to, d.rec_tracking, amodal, a.p.rec_amodel_offset, o, acx, acy, tx, ty);
    o[CT_TRK_ID] = 0.f; o[CT_TRK_AGE] = 1.f; o[CT_TRK_ACTIVE] = 0.f;
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

  // a stream runs --public_det only where the launch has the public detections (as.public_det); the association
  // scratch is present whenever a stream may run either mode
  const bool hung = so.hungarian != 0, pub = so.public_det != 0 && a.as.public_det != 0;
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
    const float new_thresh = so.new_thresh;
    const int max_age = so.max_age;
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
      if (o[CT_TRK_SCORE] > new_thresh) {
        ++ids;
        o[CT_TRK_ID] = (float)ids; o[CT_TRK_AGE] = 1.f; o[CT_TRK_ACTIVE] = 1.f;
        if (pos < T) s_pos_det[i] = pos++;
      }
    };
    auto coast = [&](int j) {
      float* t = s_old + (size_t)j * TF;
      if (t[CT_TRK_AGE] < (float)max_age) {
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
  track_boxes(d, b, trk, total, so.pre_thresh, tid);
}

// ct_track_start: stream starts[e][0] begins a new video -- Tracker.reset + init_track(seeds): its T track rows, counts
// and payload rows are cleared, its starts[e][1] seed rows (already filtered and numbered on the host) written, and its
// render boxes computed from them by the same code as the track step's.  One CTA per started stream; the seeds of
// entry e follow those of entries 0..e-1 in `seeds`.
// RESTORE (ct_track_restore): entries are (stream, n, id_count), the rows are an exported stream's verbatim (ids, ages
// and active kept) with their payload rows in `pay_rows`, and counts = (n, id_count).  A template parameter so that
// ct_track_start's instantiation stays as it was.  opts (_opts entry points): the boxes use opts[b].pre_thresh; NULL =
// the descriptor's.
template <bool RESTORE = false>
__global__ void __launch_bounds__(TRK_THREADS)
track_start_kernel(const ct_track_desc d, float* __restrict__ payload, int Wp, const int* __restrict__ starts,
                   const float* __restrict__ seeds, const float* __restrict__ pay_rows,
                   const ct_track_opts* __restrict__ opts) {
  constexpr int S = RESTORE ? 3 : 2;                          // int32 per entry
  const int e = blockIdx.x, tid = threadIdx.x, T = d.max_tracks;
  const int b = starts[S * e];
  if (b < 0 || b >= d.B) return;
  auto clamp_n = [&](int n) { return seeds == nullptr ? 0 : (n < 0 ? 0 : (n > T ? T : n)); };
  size_t off = 0;
  for (int k = 0; k < e; ++k) off += (size_t)clamp_n(starts[S * k + 1]);
  const int n = clamp_n(starts[S * e + 1]);
  float* trk = d.tracks + (size_t)b * T * TF;
  const float* src = seeds ? seeds + off * TF : nullptr;
  for (int i = tid; i < T * TF; i += TRK_THREADS) trk[i] = i < n * TF ? src[i] : 0.f;
  if (payload) {
    const float* psrc = RESTORE && pay_rows ? pay_rows + off * Wp : nullptr;
    for (int i = tid; i < T * Wp; i += TRK_THREADS) payload[(size_t)b * T * Wp + i] = psrc && i < n * Wp ? psrc[i] : 0.f;
  }
  if (tid == 0) { d.counts[b * 2 + 0] = n; d.counts[b * 2 + 1] = RESTORE ? starts[S * e + 2] : n; }
  __syncthreads();     // the seed rows written above are re-read below by other threads
  __threadfence_block();
  track_boxes(d, b, trk, n, opts ? opts[b].pre_thresh : d.pre_thresh, tid);
}

// splat of the boxes written by track_step_kernel; rows with radius < 0 are skipped.  grid = B*T (fixed: graph-capturable)
// image_of (ct_render_tracks_mapped): a row of stream s splats into image image_of[s] (< 0: skipped); NULL = identity.
template <bool MAP = false>
__global__ void render_tracks_kernel(const float* __restrict__ boxes, int n, float* __restrict__ hm, int B, int H, int W,
                                     const int* __restrict__ image_of, int n_streams) {
  const int i = blockIdx.x;
  if (i >= n) return;
  const float rf = boxes[i * 5 + 3];
  if (rf < 0.f) return;
  int b = (int)boxes[i * 5 + 0];
  const int cx = (int)boxes[i * 5 + 1], cy = (int)boxes[i * 5 + 2], r = (int)rf;
  if constexpr (MAP) {
    if (b < 0 || b >= n_streams) return;
    b = image_of[b];
  }
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

// ct_post_process: Detector.post_process + merge_outputs of runners without a tracker.  CTA i on records[i] writes
// stream b = streams[i]'s (identity without a map) kept detections: the score-sorted records with score > out_thresh
// are a prefix, each of its rows computed by det_row (+ det_payload) independently of the others.
constexpr int DET_THREADS = 128;
constexpr int DF = CT_DET_FLOATS;

struct DetArgs {
  ct_det_desc d;
  ct_track_payload p;      // read by the payload instantiation only
  const int* streams;      // NULL = identity
  int n_streams;
  const ct_track_opts* opts;   // ct_post_process_opts: stream b keeps score > opts[b].out_thresh; NULL = d.out_thresh
};

template <bool PAY>
__global__ void __launch_bounds__(DET_THREADS) post_process_kernel(const DetArgs a) {
  const ct_det_desc& d = a.d;
  const int b = a.streams ? a.streams[blockIdx.x] : (int)blockIdx.x;
  if (b < 0 || b >= a.n_streams) return;                    // a padding image, or no stream: nothing is written
  __shared__ int s_n;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  const int K = d.K, F = d.F;
  const float* rec = d.records + (size_t)blockIdx.x * K * F;
  const float out_thresh = a.opts ? a.opts[b].out_thresh : d.out_thresh;
  int cnt = 0;
  for (int i = threadIdx.x; i < K; i += DET_THREADS) cnt += rec[(size_t)i * F + CT_REC_SCORE] > out_thresh ? 1 : 0;
  atomicAdd(&s_n, cnt);
  __syncthreads();
  const int N = s_n;
  const float* to = d.trans_out_inv + b * 6;
  const bool amodal = PAY && a.p.rec_rot >= 0 && a.p.rec_dep >= 0 && a.p.rec_dim >= 0;
  const float* P = PAY && a.p.calib ? a.p.calib + b * 12 : nullptr;
  float* out = d.dets + (size_t)b * K * DF;
  for (int i = threadIdx.x; i < N; i += DET_THREADS) {
    const float* r = rec + (size_t)i * F;
    float o[DF], acx, acy, tx, ty;
    det_row(r, to, d.rec_tracking, amodal, PAY ? a.p.rec_amodel_offset : -1, o, acx, acy, tx, ty);
#pragma unroll
    for (int f = 0; f < DF; ++f) out[(size_t)i * DF + f] = o[f];
    if constexpr (PAY) det_payload(a.p, r, to, o + CT_TRK_CT, P, a.p.payload + ((size_t)b * K + i) * a.p.width);
  }
  if (threadIdx.x == 0) d.counts[b] = N;
}

// ------------------------------------------------------------------------------------------------------------------
// pre_process: cv2.warpAffine(src u8 HWC, M, (ow, oh), INTER_LINEAR, BORDER_CONSTANT 0) then (v/255 - mean)/std, CHW.
// cv2's arithmetic (imgwarp.cpp warpAffine + remapBilinear): source coordinates in 1/1024 px fixed point rounded
// to 1/32 px, bilinear weights from a 32x32 table of int16 coefficients summing to 2^15, result (sum + 2^14) >> 15.
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int sat_int(double v) {        // cv::saturate_cast<int>(double) = cvRound, ties to even
  return __double2int_rn(v);
}

__device__ __forceinline__ int sat_u8(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

// cv2.cvtColor's YUV 4:2:0 -> BGR of one pixel (COLOR_YUV2BGR_NV12 / _I420): BT.601 limited range in 20-bit fixed
// point, y = max(Y - 16, 0) * 1.164, rounded by + 2^19 before the shift.  Every sum stays below 2^30 in magnitude.
__device__ __forceinline__ void yuv_to_bgr(int Y, int U, int V, int bgr[3]) {
  const int y = max(Y - 16, 0) * 1220542 + (1 << 19), u = U - 128, v = V - 128;
  bgr[0] = sat_u8((y + 2116026 * u) >> 20);
  bgr[1] = sat_u8((y - 852492 * v - 409993 * u) >> 20);
  bgr[2] = sat_u8((y + 1673527 * v) >> 20);
}

// The warped uint8 BGR value of output pixel (x, y): src uint8 [sh, sw, 3] with row pitch sstep bytes, M the inverted
// (dst -> src) map.  The one copy of the per-pixel warp arithmetic: ct_warp_affine_normalize and the frames kernels
// all call it, so that the fused stem input is byte-identical to the fp32 image packed afterwards.
// FMT = CT_FRAME_NV12 / CT_FRAME_I420: src is the [3sh/2, sw] 4:2:0 frame (luma pitch sstep) and each tap inside the
// frame is converted to BGR first, so the result is the warp of cv2.cvtColor's BGR image; taps outside read BGR 0.
template <int FMT = CT_FRAME_BGR>
__device__ __forceinline__ void warp_bilinear_u8(const unsigned char* __restrict__ img, int sh, int sw, int sstep,
                                                 const double* M, int x, int y, int p8[3]) {
  const int AB_BITS = 10, AB_SCALE = 1 << AB_BITS, INTER_BITS = 5, INTER_TAB = 1 << INTER_BITS;
  const int round_delta = AB_SCALE / INTER_TAB / 2;
  // cv2 rounds M[1]*y and the sum + M[2] separately: the _rn intrinsics keep nvcc from fusing them into one DFMA, whose
  // single rounding moves a row term that lands on a 1/2048 px tie to the other 1/32 px step
  const int adelta = sat_int(__dmul_rn(__dmul_rn(M[0], x), AB_SCALE)), bdelta = sat_int(__dmul_rn(__dmul_rn(M[3], x), AB_SCALE));
  const int X0 = sat_int(__dmul_rn(__dadd_rn(__dmul_rn(M[1], y), M[2]), AB_SCALE)) + round_delta;
  const int Y0 = sat_int(__dmul_rn(__dadd_rn(__dmul_rn(M[4], y), M[5]), AB_SCALE)) + round_delta;
  const int X = (X0 + adelta) >> (AB_BITS - INTER_BITS), Y = (Y0 + bdelta) >> (AB_BITS - INTER_BITS);
  const int sx = X >> INTER_BITS, sy = Y >> INTER_BITS;          // arithmetic shifts: floor
  // BilinearTab_i: (1-fy|fy) x (1-fx|fx) in 1/32 steps, scaled by 2^15: exact integers (the table's one saturated
  // entry, fx = fy = 0, yields the same pixel as the exact weight 32768)
  const int fx = X & (INTER_TAB - 1), fy = Y & (INTER_TAB - 1);
  const int w[4] = {(32 - fy) * (32 - fx) * 32, (32 - fy) * fx * 32, fy * (32 - fx) * 32, fy * fx * 32};
  if constexpr (FMT == CT_FRAME_BGR) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      int acc = 0;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int yy = sy + (t >> 1), xx = sx + (t & 1);
        const int v = ((unsigned)yy < (unsigned)sh && (unsigned)xx < (unsigned)sw) ? img[(size_t)yy * sstep + xx * 3 + c] : 0;
        acc += v * w[t];
      }
      p8[c] = sat_u8((acc + (1 << 14)) >> 15);
    }
  } else {
    const unsigned char* chroma = img + (size_t)sh * sstep;
    int acc[3] = {0, 0, 0};
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int yy = sy + (t >> 1), xx = sx + (t & 1);
      if ((unsigned)yy < (unsigned)sh && (unsigned)xx < (unsigned)sw) {
        int U, V;
        if constexpr (FMT == CT_FRAME_NV12) {       // row yy/2 of interleaved U V, the pair of column xx/2
          const unsigned char* uv = chroma + (size_t)(yy >> 1) * sstep + (xx & ~1);
          U = uv[0];
          V = uv[1];
        } else {       // I420: half-row k of the chroma planes lies at (k/2) pitch + (k%2) sw/2; U = 0..sh/2-1, V after
          const int ku = yy >> 1, kv = (sh >> 1) + ku, cx = xx >> 1;
          U = chroma[(size_t)(ku >> 1) * sstep + (ku & 1) * (sw >> 1) + cx];
          V = chroma[(size_t)(kv >> 1) * sstep + (kv & 1) * (sw >> 1) + cx];
        }
        int bgr[3];
        yuv_to_bgr(img[(size_t)yy * sstep + xx], U, V, bgr);
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] += bgr[c] * w[t];
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) p8[c] = sat_u8((acc[c] + (1 << 14)) >> 15);
  }
}

// ((inp / 255. - mean) / std).astype(float32): float64 arithmetic, one final rounding
__device__ __forceinline__ float normalize_u8(int v, float mean, float stdv) {
  return (float)(((double)v / 255.0 - (double)mean) / (double)stdv);
}

// ((v / 255 - mean) / std) of a warped pixel into an fp32 CHW image: o points at channel 0, planes `plane` floats apart.
__device__ __forceinline__ void store_norm_pixel(const int p8[3], float* o, size_t plane, float3 mean, float3 stdv) {
  o[0] = normalize_u8(p8[0], mean.x, stdv.x);
  o[plane] = normalize_u8(p8[1], mean.y, stdv.y);
  o[2 * plane] = normalize_u8(p8[2], mean.z, stdv.z);
}

// One fp32 CHW output pixel (x, y) of ct_warp_affine_normalize.
__device__ __forceinline__ void warp_norm_pixel(const unsigned char* __restrict__ img, int sh, int sw, int sstep,
                                                const double* M, int x, int y, float* o, size_t plane, float3 mean,
                                                float3 stdv) {
  int p8[3];
  warp_bilinear_u8(img, sh, sw, sstep, M, x, y, p8);
  store_norm_pixel(p8, o, plane, mean, stdv);
}

__global__ void warp_affine_norm_kernel(const unsigned char* __restrict__ src, int sh, int sw, int sstep,
                                        float* __restrict__ dst, int B, int oh, int ow,
                                        const double* __restrict__ minv /*[B][6] dst->src*/, float3 mean, float3 stdv) {
  const size_t total = (size_t)B * oh * ow;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / ((size_t)oh * ow));
    const size_t r = i - (size_t)b * oh * ow;
    const int y = (int)(r / ow), x = (int)(r - (size_t)y * ow);
    const size_t plane = (size_t)oh * ow;
    warp_norm_pixel(src + (size_t)b * sh * sstep, sh, sw, sstep, minv + b * 6, x, y,
                    dst + (size_t)b * 3 * plane + (size_t)y * ow + x, plane, mean, stdv);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Where a frames kernel finds stream b's ct_frame: a device array [B] that may change between graph replays.  Each CTA
// copies its stream's descriptor to shared memory once and checks it against the buffer size, since the host cannot:
// an invalid one yields zeros and no read of the frame buffers.
// ------------------------------------------------------------------------------------------------------------------
struct DeviceFrames {
  const ct_frame* f;
  long long buf_bytes;
};

// a known format, even sizes for 4:2:0, a row pitch that holds a row, and every row read inside the buffer
__device__ __forceinline__ bool frame_in_buffer(const ct_frame& f, long long buf_bytes) {
  if (f.h <= 0 || f.w <= 0 || f.offset < 0 || f.offset > buf_bytes) return false;
  long long rows = f.h, row_bytes = 3LL * f.w;
  if (f.format == CT_FRAME_NV12 || f.format == CT_FRAME_I420) {
    if ((f.h | f.w) & 1) return false;
    rows = 3LL * (f.h / 2);
    row_bytes = f.w;
  } else if (f.format != CT_FRAME_BGR) {
    return false;
  }
  return (long long)f.step >= row_bytes && (rows - 1) * f.step + row_bytes <= buf_bytes - f.offset;
}

// The warped BGR pixel (x, y) of the frame f describes at src (its first byte), in f's format `fmt`.
__device__ __forceinline__ void warp_frame_u8(const unsigned char* __restrict__ src, const ct_frame& f, int fmt, int x,
                                              int y, int p8[3]) {
  if (fmt == CT_FRAME_NV12) return warp_bilinear_u8<CT_FRAME_NV12>(src, f.h, f.w, f.step, f.minv, x, y, p8);
  if (fmt == CT_FRAME_I420) return warp_bilinear_u8<CT_FRAME_I420>(src, f.h, f.w, f.step, f.minv, x, y, p8);
  warp_bilinear_u8(src, f.h, f.w, f.step, f.minv, x, y, p8);
}

// -> this CTA's descriptor (stream blockIdx.y) and whether it may be read; ends with __syncthreads()
__device__ __forceinline__ const ct_frame& cta_frame(const DeviceFrames& fs, ct_frame* s_f, bool& ok) {
  __shared__ int s_ok;
  if (threadIdx.x == 0) {
    *s_f = fs.f[blockIdx.y];
    s_ok = frame_in_buffer(*s_f, fs.buf_bytes);
  }
  __syncthreads();
  ok = s_ok != 0;
  return *s_f;
}

// ct_warp_frames_normalize: blockIdx.y = stream, its image by a grid-stride loop over blockIdx.x
__global__ void warp_frames_norm_kernel(const unsigned char* __restrict__ src, const __grid_constant__ DeviceFrames fs,
                                        float* __restrict__ dst, int oh, int ow, float3 mean, float3 stdv) {
  __shared__ ct_frame s_f;
  bool ok;
  const ct_frame& f = cta_frame(fs, &s_f, ok);
  const int fmt = f.format;
  const size_t plane = (size_t)oh * ow;
  float* o = dst + (size_t)blockIdx.y * 3 * plane;
  for (size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x; r < plane; r += (size_t)gridDim.x * blockDim.x) {
    const int y = (int)(r / ow), x = (int)(r - (size_t)y * ow);
    if (ok) {
      int p8[3];
      warp_frame_u8(src + f.offset, f, fmt, x, y, p8);
      store_norm_pixel(p8, o + r, plane, mean, stdv);
    } else {
      o[r] = o[r + plane] = o[r + 2 * plane] = 0.f;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// ct_pack_stem_frames_dev: the tensor-core stem's input [B,H,W,8] bf16 = (norm(warp(cur_b)) x3, norm(warp(prev_b)) x3,
// pre_hm, 0) straight from each stream's uint8 frame.  blockIdx.y = stream (its descriptor read once from device
// memory), one 16-byte output pixel per thread and iteration.  The normalisation depends on the 8-bit value only: a
// 3 x 256 table built per CTA with normalize_u8 gives the same floats without a per-pixel fp64 divide.
// FLIP (ct_pack_stem_frames_flip_dev): out is [2B,H,W,8] and image B+b is image b mirrored.  The mirrored packed pixel
// (y, W-1-x) equals the original's (y, x) in all 8 channels (frame, previous frame and pre_hm are all mirrored), so each
// pixel is warped once and its 16-byte vector stored twice.
// ------------------------------------------------------------------------------------------------------------------
constexpr int PACK_THREADS = 256;
constexpr int PACK_PIX_PER_THREAD = 4;      // pixels per thread: amortises the table build over 1024 pixels per CTA

// The PACK_PIX_PER_THREAD output pixels of one thread, frame format FMT (uniform over the CTA, so each format's loop
// is a code region of its own and a BGR stream runs the BGR-only loop)
template <bool FLIP, int FMT>
__device__ __forceinline__ void pack_pixels(const unsigned char* __restrict__ src, const unsigned char* __restrict__ psrc,
                                            const ct_frame& f, bool ok, const float (*tab)[256], int b, int B,
                                            size_t base, const float* __restrict__ hm, uint4* __restrict__ out, int H,
                                            int W) {
  const size_t plane = (size_t)H * W;
#pragma unroll
  for (int k = 0; k < PACK_PIX_PER_THREAD; ++k) {
    const size_t r = base + (size_t)k * PACK_THREADS;
    if (r >= plane) break;
    const int y = (int)(r / W), x = (int)(r - (size_t)y * W);
    uint4 o = make_uint4(0u, 0u, 0u, 0u);
    if (ok) {
      float v[8];
      int p8[3];
      warp_bilinear_u8<FMT>(src, f.h, f.w, f.step, f.minv, x, y, p8);
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = tab[c][p8[c]];
      if (psrc) {
        warp_bilinear_u8<FMT>(psrc, f.h, f.w, f.step, f.minv, x, y, p8);
#pragma unroll
        for (int c = 0; c < 3; ++c) v[3 + c] = tab[c][p8[c]];
      } else {
        v[3] = v[4] = v[5] = 0.f;
      }
      v[6] = hm ? __ldg(hm + (size_t)b * plane + r) : 0.f;
      v[7] = 0.f;
      __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
      for (int q = 0; q < 4; ++q) h[q] = __floats2bfloat162_rn(v[2 * q], v[2 * q + 1]);
    }
    out[(size_t)b * plane + r] = o;
    if constexpr (FLIP) out[(size_t)(B + b) * plane + (size_t)y * W + (W - 1 - x)] = o;
  }
}

// 6 CTAs per SM, at most 40 registers -- the occupancy of the BGR-only sampler's 36 (allocated in steps of 8); without
// the bound the YUV samplers take the flip form to 48 registers and 5 CTAs.
constexpr int PACK_DEV_MIN_CTAS = 6;

template <bool FLIP>
__global__ void __launch_bounds__(PACK_THREADS, PACK_DEV_MIN_CTAS)
pack_stem_frames_dev_kernel(const unsigned char* __restrict__ cur, const unsigned char* __restrict__ prev,
                            const __grid_constant__ DeviceFrames fs, float3 mean, float3 stdv,
                            const float* __restrict__ hm, uint4* __restrict__ out, int H, int W) {
  __shared__ float tab[3][256];
  __shared__ ct_frame s_f;
  for (int i = threadIdx.x; i < 3 * 256; i += PACK_THREADS) {
    const int c = i >> 8, v = i & 255;
    tab[c][v] = normalize_u8(v, c == 0 ? mean.x : (c == 1 ? mean.y : mean.z), c == 0 ? stdv.x : (c == 1 ? stdv.y : stdv.z));
  }
  bool ok;
  const ct_frame& f = cta_frame(fs, &s_f, ok);
  const int b = blockIdx.y, B = gridDim.y;
  const unsigned char* src = cur + f.offset;
  const unsigned char* psrc = prev ? prev + f.offset : nullptr;
  const size_t base = (size_t)blockIdx.x * PACK_THREADS * PACK_PIX_PER_THREAD + threadIdx.x;
  const int fmt = f.format;
  if (fmt == CT_FRAME_NV12)
    return pack_pixels<FLIP, CT_FRAME_NV12>(src, psrc, f, ok, tab, b, B, base, hm, out, H, W);
  if (fmt == CT_FRAME_I420)
    return pack_pixels<FLIP, CT_FRAME_I420>(src, psrc, f, ok, tab, b, B, base, hm, out, H, W);
  pack_pixels<FLIP, CT_FRAME_BGR>(src, psrc, f, ok, tab, b, B, base, hm, out, H, W);
}

// ------------------------------------------------------------------------------------------------------------------
// ct_stage_frames: each stream's device frame copied into its region of a frame slot, in the slot's layout.
// blockIdx.y = stream, one warp per destination row, the frame's rows spread over blockIdx.x.  A row whose source and
// destination rows are 16-byte aligned moves 16 bytes per lane and access (the RGB -> BGR swap and the planar ->
// interleaved transpose work on 16 pixels = 48 bytes in registers); unaligned rows and the end of a row go byte by byte.
// A pure copy: HBM-bound.
// ------------------------------------------------------------------------------------------------------------------
constexpr int STAGE_THREADS = 256;
constexpr int STAGE_WARPS = STAGE_THREADS / 32;

struct StageFrame {
  const unsigned char* src[3];
  long long pitch[3];
  long long offset;           // destination
  int h, w, step, layout;
};

struct StageArgs {
  StageFrame f[CT_FRAMES_PER_LAUNCH];
};

__device__ __forceinline__ bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

// byte j of the little-endian words v
__device__ __forceinline__ uint32_t byte_at(const uint32_t* v, int j) { return (v[j >> 2] >> (8 * (j & 3))) & 0xffu; }

// d[0, n) <- s[0, n) by one warp: 16-byte accesses when s and d share their alignment
__device__ __forceinline__ void stage_copy(const unsigned char* __restrict__ s, unsigned char* __restrict__ d, int n,
                                           int lane) {
  int head = n, body = 0;
  if ((((uintptr_t)s ^ (uintptr_t)d) & 15) == 0) {
    head = min((int)((16 - ((uintptr_t)d & 15)) & 15), n);
    body = (n - head) >> 4;
    const uint4* sv = reinterpret_cast<const uint4*>(s + head);
    uint4* dv = reinterpret_cast<uint4*>(d + head);
    for (int i = lane; i < body; i += 32) dv[i] = __ldg(sv + i);
  }
  for (int i = lane; i < head; i += 32) d[i] = s[i];
  for (int i = head + (body << 4) + lane; i < n; i += 32) d[i] = s[i];
}

// One BGR row of w pixels from interleaved RGB (PLANAR = false: s0) or from the R, G, B rows s0, s1, s2.  Output byte
// j = 3x + c takes source byte 3x + 2 - c, or byte x of plane 2 - c.
template <bool PLANAR>
__device__ __forceinline__ void stage_bgr_row(const unsigned char* __restrict__ s0, const unsigned char* __restrict__ s1,
                                              const unsigned char* __restrict__ s2, unsigned char* __restrict__ d, int w,
                                              int lane) {
  int done = 0;
  if (aligned16(s0) && aligned16(d) && (!PLANAR || (aligned16(s1) && aligned16(s2)))) {
    done = w >> 4;                                          // chunks of 16 pixels
    for (int c = lane; c < done; c += 32) {
      uint32_t in[12], out[12];
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const unsigned char* sq = !PLANAR ? s0 : (q == 0 ? s0 : (q == 1 ? s1 : s2));
        const uint4 t = __ldg(reinterpret_cast<const uint4*>(sq) + (PLANAR ? c : 3 * c + q));
        in[4 * q] = t.x, in[4 * q + 1] = t.y, in[4 * q + 2] = t.z, in[4 * q + 3] = t.w;
      }
#pragma unroll
      for (int k = 0; k < 12; ++k) {
        uint32_t o = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int j = 4 * k + i, x = j / 3, ch = j % 3;
          o |= byte_at(in, PLANAR ? (2 - ch) * 16 + x : 3 * x + 2 - ch) << (8 * i);
        }
        out[k] = o;
      }
      uint4* dv = reinterpret_cast<uint4*>(d) + 3 * c;
#pragma unroll
      for (int q = 0; q < 3; ++q) dv[q] = make_uint4(out[4 * q], out[4 * q + 1], out[4 * q + 2], out[4 * q + 3]);
    }
    done <<= 4;
  }
  for (int j = 3 * done + lane; j < 3 * w; j += 32) {
    const int x = j / 3, ch = j - 3 * x;
    d[j] = !PLANAR ? s0[3 * x + 2 - ch] : (ch == 0 ? s2[x] : (ch == 1 ? s1[x] : s0[x]));
  }
}

__global__ void __launch_bounds__(STAGE_THREADS)
stage_frames_kernel(const __grid_constant__ StageArgs a, unsigned char* __restrict__ buf) {
  const StageFrame& f = a.f[blockIdx.y];
  const int h = f.h, w = f.w, step = f.step, layout = f.layout, lane = threadIdx.x & 31;
  const unsigned char *src0 = f.src[0], *src1 = f.src[1], *src2 = f.src[2];
  const long long p0 = f.pitch[0], p1 = f.pitch[1], p2 = f.pitch[2];
  const int rows = layout == CT_SRC_NV12 ? h + h / 2 : (layout == CT_SRC_I420 ? 2 * h : h);
  unsigned char* dst = buf + f.offset;
  for (int r = blockIdx.x * STAGE_WARPS + (threadIdx.x >> 5); r < rows; r += gridDim.x * STAGE_WARPS) {
    unsigned char* d = dst + (size_t)r * step;
    if (layout == CT_SRC_RGB) {
      stage_bgr_row<false>(src0 + r * p0, nullptr, nullptr, d, w, lane);
      continue;
    }
    if (layout == CT_SRC_RGB_PLANAR) {
      stage_bgr_row<true>(src0 + r * p0, src1 + r * p1, src2 + r * p2, d, w, lane);
      continue;
    }
    // a plain copy: a BGR row, a luma row, an NV12 UV row or an I420 chroma half-row
    const unsigned char* s = src0 + r * p0;
    int n = layout == CT_SRC_BGR ? 3 * w : w;
    if (layout != CT_SRC_BGR && r >= h) {
      const int k = r - h, hh = h >> 1;
      if (layout == CT_SRC_NV12) {
        s = src1 + k * p1;
      } else {   // I420 half-row k: U rows 0..h/2-1, then V; two half-rows to a destination row, as cv2 lays them out
        s = k < hh ? src1 + k * p1 : src2 + (k - hh) * p2;
        d = dst + (size_t)(h + (k >> 1)) * step + (k & 1) * (w >> 1);
        n = w >> 1;
      }
    }
    stage_copy(s, d, n, lane);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// ct_crop_boxes: crop k of stream b = cv2.warpAffine(frame_b, M, (out_w, out_h), INTER_LINEAR | WARP_INVERSE_MAP,
// BORDER_CONSTANT 0) with the box's dst -> src map M = [sx, 0, (x0 - .5) + .5 sx, 0, sy, (y0 - .5) + .5 sy],
// sx = (x1 - x0) / out_w, sy = (y1 - y0) / out_h in fp64, each step rounded on its own (no FMA contraction).  The taps
// are warp_bilinear_u8's, so a 4:2:0 frame gives the crop of its cv2.cvtColor BGR image.
// grid (pixel chunks, K, n): CTA (., k, i) writes crop k of image i's stream and exits when k is past its count, so the
// launch shape depends on n, K and the crop size alone.  A CTA's CROP_PIX * CROP_THREADS consecutive crop pixels are
// warped with adjacent pixels on adjacent lanes (their taps are neighbours: coalesced loads), staged as bytes in shared
// memory, and stored as 16-byte vectors on adjacent lanes where the crop is 16-byte aligned.  Its time goes to the
// taps, not to the writes (DESIGN §5).
// ------------------------------------------------------------------------------------------------------------------
constexpr int CROP_THREADS = 128;
constexpr int CROP_PIX = 16;                // pixels per thread
constexpr int CROP_CTA_BYTES = 3 * CROP_PIX * CROP_THREADS;
constexpr float CROP_MAX_COORD = 16384.f;   // beyond it cv2's int16 source map would saturate: the crop is zeros

struct CropArgs {
  ct_crop_desc d;
  const int* streams;      // NULL = identity
  int n_streams;
  ct_crop_tensor t;        // ct_crop_boxes_tensor's output (the tensor forms)
};

// Output forms of crop_boxes_kernel: ct_crop_boxes' uint8 BGR crops, or ct_crop_boxes_tensor's packed NCHW rows of
// one ct_crop_type.
constexpr int CROP_U8 = -1;

// Which rows of stream b image i's crops come from, shared by both entry points: the first counts[b] rows, clamped to
// [0, min(K, rows_per_stream)], none for an invalid frame (nothing is read); with a track table, cut at the first of
// them whose active column is 0 (crop_row_inactive).
__device__ __forceinline__ int crop_row_limit(const ct_crop_desc& d, const ct_frame& f, int b) {
  const int n = d.counts[(size_t)b * d.counts_stride];
  return frame_in_buffer(f, d.buf_bytes) ? max(0, min(n, min(d.K, d.rows_per_stream))) : 0;
}
__device__ __forceinline__ const float* crop_rows(const ct_crop_desc& d, int b) {
  return d.rows + (size_t)b * d.rows_per_stream * d.row_floats;
}
__device__ __forceinline__ bool crop_row_inactive(const ct_crop_desc& d, const float* rows, int r) {
  return rows[(size_t)r * d.row_floats + d.active_col] == 0.f;
}

// The CTA's pixels [p0, p0 + CROP_PIX * CROP_THREADS) of the crop -> s_px (3 bytes each); zero = the box failed the
// guard (an all-zero crop).
template <int FMT>
__device__ __forceinline__ void crop_pixels(const unsigned char* __restrict__ src, const ct_frame& f, const double* M,
                                            bool zero, int out_w, size_t total, size_t p0, unsigned char* s_px) {
#pragma unroll 4
  for (int q = 0; q < CROP_PIX; ++q) {
    const int j = q * CROP_THREADS + (int)threadIdx.x;
    const size_t p = p0 + j;
    if (p >= total) break;
    int p8[3] = {0, 0, 0};
    if (!zero) {
      const int y = (int)(p / out_w), x = (int)(p - (size_t)y * out_w);
      warp_bilinear_u8<FMT>(src, f.h, f.w, f.step, M, x, y, p8);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) s_px[3 * j + c] = (unsigned char)p8[c];
  }
}

// The CTA's npx staged pixels s_px -> the uint8 BGR crop at dst (crop pixel p0).
__device__ __forceinline__ void crop_store_u8(const unsigned char* s_px, unsigned char* dst, int npx) {
  const int nbytes = 3 * npx;
  if (aligned16(dst)) {                                     // p0 * 3 is a multiple of 16: aligned when the crop is
    const int vec = nbytes >> 4;
    for (int j = threadIdx.x; j < vec; j += CROP_THREADS)
      reinterpret_cast<uint4*>(dst)[j] = reinterpret_cast<const uint4*>(s_px)[j];
    for (int j = (vec << 4) + threadIdx.x; j < nbytes; j += CROP_THREADS) dst[j] = s_px[j];
  } else {
    for (int j = threadIdx.x; j < nbytes; j += CROP_THREADS) dst[j] = s_px[j];
  }
}

// The element bits of value v in the output type TYPE (round to nearest even), in the low bits of a word.
template <int TYPE>
__device__ __forceinline__ uint32_t crop_elem_bits(float v) {
  if constexpr (TYPE == CT_CROP_F32) return __float_as_uint(v);
  else if constexpr (TYPE == CT_CROP_F16) return __half_as_ushort(__float2half_rn(v));
  else return __bfloat16_as_ushort(__float2bfloat16_rn(v));
}

// The CTA's npx staged pixels s_px -> row's three channel planes (row: out + row index * 3 * total elements), from
// crop pixel p0.  Element (c, byte u) = ((float)u / 255 - mean[c]) / std[c], each operation an fp32 rounding of its
// own, then rounded into TYPE: a table of the 3 x 256 values per CTA, so the pixels cost one shared load each.  Each
// plane's run is stored as 16-byte vectors from its first 16-byte boundary on, the elements around them one by one.
template <int TYPE>
__device__ __forceinline__ void crop_store_tensor(const ct_crop_tensor& t, const unsigned char* s_px, void* row,
                                                  size_t total, size_t p0, int npx) {
  using T = typename std::conditional<TYPE == CT_CROP_F32, uint32_t, uint16_t>::type;
  constexpr int V = 16 / (int)sizeof(T);
  __shared__ uint32_t s_lut[3][256];
  for (int j = threadIdx.x; j < 3 * 256; j += CROP_THREADS) {
    const int c = j >> 8;
    s_lut[c][j & 255] = crop_elem_bits<TYPE>(__fdiv_rn(__fsub_rn(__fdiv_rn((float)(j & 255), 255.f), t.mean[c]), t.std[c]));
  }
  __syncthreads();
#pragma unroll 1
  for (int c = 0; c < 3; ++c) {
    const int sc = t.order == CT_CROP_RGB ? 2 - c : c;    // the staged pixels are BGR
    const uint32_t* lut = s_lut[c];
    const unsigned char* px = s_px + sc;
    T* dst = reinterpret_cast<T*>(row) + (size_t)c * total + p0;
    const int head = min(npx, (int)(((16 - ((uintptr_t)dst & 15)) & 15) / sizeof(T)));
    const int vec = (npx - head) / V;
    for (int j = threadIdx.x; j < head; j += CROP_THREADS) dst[j] = (T)lut[px[3 * j]];
    for (int j = threadIdx.x; j < vec; j += CROP_THREADS) {
      const int q = head + j * V;
      uint32_t w[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if constexpr (V == 4) w[e] = lut[px[3 * (q + e)]];
        else w[e] = lut[px[3 * (q + 2 * e)]] | (lut[px[3 * (q + 2 * e + 1)]] << 16);
      }
      *reinterpret_cast<uint4*>(dst + q) = make_uint4(w[0], w[1], w[2], w[3]);
    }
    for (int j = head + vec * V + threadIdx.x; j < npx; j += CROP_THREADS) dst[j] = (T)lut[px[3 * j]];
  }
}

// FORM CROP_U8 (ct_crop_boxes): crop k of stream b -> out[b][k], its count -> out_counts[b] (the row selection here).
// FORM a ct_crop_type (ct_crop_boxes_tensor): the stream's rows and count come from t.out_offsets, which
// crop_offsets_kernel wrote with the same row selection just before; crop k -> row out_offsets[b] + k of t.out.
template <int FORM>
__global__ void __launch_bounds__(CROP_THREADS) crop_boxes_kernel(const __grid_constant__ CropArgs a) {
  const ct_crop_desc& d = a.d;
  const int i = blockIdx.z, k = blockIdx.y;
  const int b = a.streams ? a.streams[i] : i;
  if (b < 0 || b >= a.n_streams) return;                    // a padding image, or no stream: nothing is written
  __shared__ ct_frame s_f;
  __shared__ int s_cnt, s_first;
  const float* rows = crop_rows(d, b);
  int n;
  if constexpr (FORM == CROP_U8) {
    if (threadIdx.x == 0) {
      s_f = d.frames[i];
      s_cnt = s_first = crop_row_limit(d, s_f, b);          // an invalid frame: no crop, nothing read
    }
    __syncthreads();
    n = s_cnt;
    if (d.active_col >= 0) {                                // track tables: the leading active rows
      for (int r = threadIdx.x; r < n; r += CROP_THREADS)
        if (crop_row_inactive(d, rows, r)) atomicMin(&s_first, r);
      __syncthreads();
      n = s_first;
    }
    if (blockIdx.x == 0 && k == 0 && threadIdx.x == 0) d.out_counts[b] = n;
  } else {
    if (threadIdx.x == 0) {
      s_f = d.frames[i];
      s_first = a.t.out_offsets[b];
      s_cnt = a.t.out_offsets[b + 1] - s_first;
    }
    __syncthreads();
    n = s_cnt;
  }
  if (k >= n) return;
  const float* bx = rows + (size_t)k * d.row_floats + CT_TRK_BBOX;
  const float x0 = bx[0], y0 = bx[1], x1 = bx[2], y1 = bx[3];
  const bool zero = !(fabsf(x0) <= CROP_MAX_COORD && fabsf(y0) <= CROP_MAX_COORD && fabsf(x1) <= CROP_MAX_COORD &&
                      fabsf(y1) <= CROP_MAX_COORD);            // non-finite or too far out
  const double sx = __ddiv_rn(__dsub_rn((double)x1, (double)x0), (double)d.out_w);
  const double sy = __ddiv_rn(__dsub_rn((double)y1, (double)y0), (double)d.out_h);
  const double M[6] = {sx, 0.0, __dadd_rn(__dsub_rn((double)x0, 0.5), __dmul_rn(0.5, sx)),
                       0.0, sy, __dadd_rn(__dsub_rn((double)y0, 0.5), __dmul_rn(0.5, sy))};
  const size_t total = (size_t)d.out_h * d.out_w;
  const size_t p0 = (size_t)blockIdx.x * CROP_THREADS * CROP_PIX;
  if (p0 >= total) return;
  __shared__ __align__(16) unsigned char s_px[CROP_CTA_BYTES];
  const ct_frame& f = s_f;
  const unsigned char* src = d.buf + f.offset;
  if (f.format == CT_FRAME_NV12) crop_pixels<CT_FRAME_NV12>(src, f, M, zero, d.out_w, total, p0, s_px);
  else if (f.format == CT_FRAME_I420) crop_pixels<CT_FRAME_I420>(src, f, M, zero, d.out_w, total, p0, s_px);
  else crop_pixels<CT_FRAME_BGR>(src, f, M, zero, d.out_w, total, p0, s_px);
  __syncthreads();
  const int npx = (int)(total - p0 < (size_t)CROP_PIX * CROP_THREADS ? total - p0 : (size_t)CROP_PIX * CROP_THREADS);
  if constexpr (FORM == CROP_U8) {
    crop_store_u8(s_px, d.out + (((size_t)b * d.K + k) * total + p0) * 3, npx);
  } else {
    const size_t row = (size_t)s_first + k;
    char* out = static_cast<char*>(a.t.out) + row * 3 * total * (FORM == CT_CROP_F32 ? 4 : 2);
    crop_store_tensor<FORM>(a.t, s_px, out, total, p0, npx);
  }
}

// ct_crop_boxes_tensor's row offsets, one CTA: stream b's crop count (crop_row_limit, cut at the first inactive row by
// one warp's ballots) -> out_counts[b], then the exclusive prefix over streams 0 .. n_streams -> t.out_offsets (a
// stream no image maps to counts 0).  Images sharing a stream are not supported (as in ct_crop_boxes).
constexpr int CROP_OFF_THREADS = 1024;

__global__ void __launch_bounds__(CROP_OFF_THREADS) crop_offsets_kernel(const __grid_constant__ CropArgs a, int n) {
  const ct_crop_desc& d = a.d;
  int* off = a.t.out_offsets;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int b = threadIdx.x; b <= a.n_streams; b += CROP_OFF_THREADS) off[b] = 0;
  __syncthreads();
  for (int i = warp; i < n; i += CROP_OFF_THREADS / 32) {   // one warp per image; every branch is warp-uniform
    const int b = a.streams ? a.streams[i] : i;
    if (b < 0 || b >= a.n_streams) continue;
    int cnt = crop_row_limit(d, d.frames[i], b);
    if (d.active_col >= 0) {
      const float* rows = crop_rows(d, b);
      for (int r0 = 0; r0 < cnt; r0 += 32) {
        const unsigned m = __ballot_sync(0xffffffffu, r0 + lane < cnt && crop_row_inactive(d, rows, r0 + lane));
        if (m) {
          cnt = r0 + __ffs(m) - 1;
          break;
        }
      }
    }
    if (lane == 0) off[b] = d.out_counts[b] = cnt;
  }
  __syncthreads();
  __shared__ int s_warp[CROP_OFF_THREADS / 32];
  int carry = 0;
  for (int b0 = 0; b0 <= a.n_streams; b0 += CROP_OFF_THREADS) {
    const int b = b0 + threadIdx.x;
    const int v = b <= a.n_streams ? off[b] : 0;
    int x = v;                                              // inclusive scan: lanes, then warps
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, s);
      if (lane >= s) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int w = s_warp[lane];
#pragma unroll
      for (int s = 1; s < 32; s <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, w, s);
        if (lane >= s) w += y;
      }
      s_warp[lane] = w;
    }
    __syncthreads();
    if (b <= a.n_streams) off[b] = carry + (warp ? s_warp[warp - 1] : 0) + x - v;
    carry += s_warp[CROP_OFF_THREADS / 32 - 1];
    __syncthreads();
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

// The payload descriptor of an F-float record: its fields inside the record, its width their sum, calib for 3D sets.
static int payload_check(const ct_track_payload* p, int32_t F) {
  CT_REQUIRE(p->payload, "null payload table");
  CT_REQUIRE(rec_field_ok(p->rec_hps, p->hps_floats, F) && (p->rec_hps < 0 || p->hps_floats % 2 == 0) &&
             rec_field_ok(p->rec_dep, 1, F) && rec_field_ok(p->rec_dim, 3, F) &&
             rec_field_ok(p->rec_rot, 8, F) && rec_field_ok(p->rec_amodel_offset, 2, F) &&
             rec_field_ok(p->rec_velocity, p->velocity_floats, F) &&
             rec_field_ok(p->rec_nuscenes_att, p->att_floats, F), "payload field outside the record");
  const bool ddd = p->rec_rot >= 0 && p->rec_dep >= 0 && p->rec_dim >= 0;
  const int64_t w = (p->rec_hps >= 0 ? p->hps_floats : 0) + (p->rec_dep >= 0 ? 1 : 0) + (p->rec_dim >= 0 ? 3 : 0) +
                    (p->rec_rot >= 0 ? 1 : 0) + (ddd ? 4 : 0) + (p->rec_velocity >= 0 ? p->velocity_floats : 0) +
                    (p->rec_nuscenes_att >= 0 ? p->att_floats : 0);
  CT_REQUIRE(w > 0 && p->width == w, "payload width does not match its fields");
  CT_REQUIRE(!ddd || p->calib, "rot, dep and dim need calib");
  return CT_OK;
}

// One track step launch: CTA i on records[i] and stream streams[i] (streams == NULL: stream i of d->B).  opts == NULL:
// every stream runs the descriptor's scalars with as's modes; else stream b runs opts[b], the association scratch is
// always present, and as->public_det says whether the launch has public detections.
static int track_step_launch(const ct_track_desc* d, const ct_track_assoc* as, const ct_track_payload* p,
                             const ct_track_opts* opts, const int32_t* streams, int32_t n_streams, void* stream) {
  CT_REQUIRE(d && as && d->records && d->trans_out_inv && d->tracks && d->counts, "null pointer");
  CT_REQUIRE(d->B > 0 && d->K > 0 && d->F >= CT_REC_HEADS && d->max_tracks >= d->K, "bad shape");
  CT_REQUIRE(d->rec_tracking < 0 || d->rec_tracking + 2 <= d->F, "tracking offset outside the record");
  CT_REQUIRE(d->boxes == nullptr || (d->trans_input != nullptr && d->inp_h > 0 && d->inp_w > 0), "boxes need trans_input");
  CT_REQUIRE(!as->public_det || (as->public_ct && as->public_n), "public_det needs public_ct and public_n");
  CT_REQUIRE(!as->public_det || as->max_public > 0, "public_det needs max_public > 0");
  if (p) {
    const int rc = payload_check(p, d->F);
    if (rc != CT_OK) return rc;
  }
  const bool scratch = opts || as->hungarian || as->public_det;
  const size_t smem = (size_t)ct_track_payload_smem_bytes(d->K, d->max_tracks, p ? p->width : 0, scratch);
  CT_REQUIRE(smem <= 200 * 1024, "track table does not fit in shared memory (lower max_tracks)");
  auto kernel = streams ? (p ? track_step_kernel<true, true> : track_step_kernel<false, true>)
                        : (p ? track_step_kernel<true> : track_step_kernel<false>);
  if (smem > 48 * 1024)
    CT_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  TrackArgs a = {};
  a.d = *d;
  a.as = *as;
  if (p) a.p = *p;
  a.pay_smem = (int)(trk_base_bytes(d->K, d->max_tracks) +
                     (scratch ? ct_track_assoc_smem_bytes(d->K, d->max_tracks) - ct_track_smem_bytes(d->K, d->max_tracks)
                              : 0));
  a.streams = streams;
  a.n_streams = n_streams;
  a.opts = opts;
  a.dflt = {d->out_thresh, d->new_thresh, d->pre_thresh, d->max_age, as->hungarian, as->public_det, {0, 0}};
  kernel<<<d->B, TRK_THREADS, smem, (cudaStream_t)stream>>>(a);
  return after_launch();
}

extern "C" int ct_track_step_payload(const ct_track_desc* d, const ct_track_assoc* as, const ct_track_payload* p,
                                     void* stream) {
  return track_step_launch(d, as, p, nullptr, nullptr, 0, stream);
}

extern "C" int ct_track_step_mapped(const ct_track_desc* d, const ct_track_assoc* as, const ct_track_payload* p,
                                    const int32_t* streams, int32_t n_streams, void* stream) {
  CT_REQUIRE(streams, "null stream map");
  CT_REQUIRE(n_streams > 0, "n_streams <= 0");
  const ct_track_assoc greedy = {};
  return track_step_launch(d, as ? as : &greedy, p, nullptr, streams, n_streams, stream);
}

extern "C" int ct_track_step_opts(const ct_track_desc* d, const ct_track_assoc* as, const ct_track_payload* p,
                                  const ct_track_opts* opts, const int32_t* streams, int32_t n_streams, void* stream) {
  CT_REQUIRE(opts, "null opts");
  CT_REQUIRE(n_streams >= 0, "n_streams < 0");
  CT_REQUIRE(!streams || n_streams > 0, "a stream map needs n_streams > 0");
  const ct_track_assoc greedy = {};
  return track_step_launch(d, as ? as : &greedy, p, opts, streams, n_streams, stream);
}

extern "C" int ct_track_step_assoc(const ct_track_desc* d, const ct_track_assoc* as, void* stream) {
  return ct_track_step_payload(d, as, nullptr, stream);
}

extern "C" int ct_track_step(const ct_track_desc* d, void* stream) {
  const ct_track_assoc greedy = {};
  return ct_track_step_assoc(d, &greedy, stream);
}

// ct_track_start / ct_track_restore (RESTORE) and their _opts forms: one CTA per entry.
template <bool RESTORE>
static int track_start_launch(const ct_track_desc* d, const ct_track_payload* p, const ct_track_opts* opts,
                              const int32_t* entries, int32_t n, const float* rows, const float* payload_rows,
                              void* stream) {
  CT_REQUIRE(d && d->tracks && d->counts, "null pointer");
  CT_REQUIRE(d->B > 0 && d->max_tracks > 0, "bad shape");
  CT_REQUIRE(d->boxes == nullptr || (d->trans_input != nullptr && d->inp_h > 0 && d->inp_w > 0), "boxes need trans_input");
  if (RESTORE) {
    CT_REQUIRE(n >= 0 && n <= d->B, "n_entries outside [0, B]");
    CT_REQUIRE(n == 0 || entries, "null entry list");
  } else {
    CT_REQUIRE(n >= 0 && n <= d->B, "n_starts outside [0, B]");
    CT_REQUIRE(n == 0 || entries, "null start list");
  }
  CT_REQUIRE(!p || (p->payload && p->width > 0), "payload table needs payload and width > 0");
  if (n == 0) return CT_OK;
  track_start_kernel<RESTORE><<<n, TRK_THREADS, 0, (cudaStream_t)stream>>>(
      *d, p ? p->payload : nullptr, p ? p->width : 0, entries, rows, payload_rows, opts);
  return after_launch();
}

extern "C" int ct_track_start(const ct_track_desc* d, const ct_track_payload* p, const int32_t* starts,
                              int32_t n_starts, const float* seeds, void* stream) {
  return track_start_launch<false>(d, p, nullptr, starts, n_starts, seeds, nullptr, stream);
}

extern "C" int ct_track_restore(const ct_track_desc* d, const ct_track_payload* p, const int32_t* entries,
                                int32_t n_entries, const float* rows, const float* payload_rows, void* stream) {
  return track_start_launch<true>(d, p, nullptr, entries, n_entries, rows, payload_rows, stream);
}

extern "C" int ct_track_start_opts(const ct_track_desc* d, const ct_track_payload* p, const ct_track_opts* opts,
                                   const int32_t* starts, int32_t n_starts, const float* seeds, void* stream) {
  CT_REQUIRE(opts, "null opts");
  return track_start_launch<false>(d, p, opts, starts, n_starts, seeds, nullptr, stream);
}

extern "C" int ct_track_restore_opts(const ct_track_desc* d, const ct_track_payload* p, const ct_track_opts* opts,
                                     const int32_t* entries, int32_t n_entries, const float* rows,
                                     const float* payload_rows, void* stream) {
  CT_REQUIRE(opts, "null opts");
  return track_start_launch<true>(d, p, opts, entries, n_entries, rows, payload_rows, stream);
}

static int post_process_launch(const ct_det_desc* d, const ct_track_payload* p, const ct_track_opts* opts,
                               const int32_t* streams, int32_t n_streams, void* stream) {
  CT_REQUIRE(d && d->records && d->trans_out_inv && d->dets && d->counts, "null pointer");
  CT_REQUIRE(d->n > 0 && d->K > 0 && d->F >= CT_REC_HEADS, "bad shape (n > 0, K > 0, F >= CT_REC_HEADS)");
  CT_REQUIRE(d->rec_tracking < 0 || (d->rec_tracking >= CT_REC_HEADS && d->rec_tracking + 2 <= d->F),
             "tracking offset outside the record");
  CT_REQUIRE(n_streams > 0, "n_streams <= 0");
  CT_REQUIRE(streams || d->n <= n_streams, "without a stream map every image needs a stream (n <= n_streams)");
  if (p) {
    const int rc = payload_check(p, d->F);
    if (rc != CT_OK) return rc;
  }
  DetArgs a = {};
  a.d = *d;
  if (p) a.p = *p;
  a.streams = streams;
  a.n_streams = n_streams;
  a.opts = opts;
  auto kernel = p ? post_process_kernel<true> : post_process_kernel<false>;
  kernel<<<d->n, DET_THREADS, 0, (cudaStream_t)stream>>>(a);
  return after_launch();
}

extern "C" int ct_post_process(const ct_det_desc* d, const ct_track_payload* p, const int32_t* streams,
                               int32_t n_streams, void* stream) {
  return post_process_launch(d, p, nullptr, streams, n_streams, stream);
}

extern "C" int ct_post_process_opts(const ct_det_desc* d, const ct_track_payload* p, const ct_track_opts* opts,
                                    const int32_t* streams, int32_t n_streams, void* stream) {
  CT_REQUIRE(opts, "null opts");
  return post_process_launch(d, p, opts, streams, n_streams, stream);
}

extern "C" int ct_render_tracks(const float* boxes, int32_t n, float* pre_hm, int32_t B, int32_t H, int32_t W,
                                void* stream) {
  CT_REQUIRE(pre_hm && boxes && n > 0, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  CT_CUDA_OK(cudaMemsetAsync(pre_hm, 0, (size_t)B * H * W * sizeof(float), st));
  render_tracks_kernel<<<n, 128, 0, st>>>(boxes, n, pre_hm, B, H, W, nullptr, 0);
  return after_launch();
}

extern "C" int ct_render_tracks_mapped(const float* boxes, int32_t n, const int32_t* image_of, int32_t n_streams,
                                       float* pre_hm, int32_t n_images, int32_t H, int32_t W, void* stream) {
  CT_REQUIRE(pre_hm && boxes && image_of && n > 0, "null pointer");
  CT_REQUIRE(n_streams > 0 && n_images > 0 && H > 0 && W > 0, "bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  CT_CUDA_OK(cudaMemsetAsync(pre_hm, 0, (size_t)n_images * H * W * sizeof(float), st));
  render_tracks_kernel<true><<<n, 128, 0, st>>>(boxes, n, pre_hm, n_images, H, W, image_of, n_streams);
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
static int pack_stem_frames_dev(const uint8_t* cur, const uint8_t* prev, const ct_frame* frames_dev, int32_t B,
                                int64_t buf_bytes, const float* mean, const float* std, const float* pre_hm, void* out,
                                int32_t H, int32_t W, void* stream) {
  CT_REQUIRE(cur && frames_dev && mean && std && out, "null pointer");
  CT_REQUIRE(B > 0 && B <= 65535 && H > 0 && W > 0, "bad shape");
  CT_REQUIRE(buf_bytes >= 0, "buf_bytes < 0");
  const size_t plane = (size_t)H * W;
  const size_t per_cta = (size_t)PACK_THREADS * PACK_PIX_PER_THREAD;
  CT_REQUIRE((plane + per_cta - 1) / per_cta <= 0x7fffffffu, "output too large");
  const DeviceFrames fs = {frames_dev, (long long)buf_bytes};
  dim3 grid((unsigned)((plane + per_cta - 1) / per_cta), (unsigned)B);
  pack_stem_frames_dev_kernel<FLIP><<<grid, PACK_THREADS, 0, (cudaStream_t)stream>>>(
      cur, prev, fs, make_float3(mean[0], mean[1], mean[2]), make_float3(std[0], std[1], std[2]), pre_hm,
      (uint4*)out, H, W);
  return after_launch();
}

extern "C" int ct_pack_stem_frames_dev(const uint8_t* cur, const uint8_t* prev, const ct_frame* frames_dev, int32_t B,
                                       int64_t buf_bytes, const float* mean, const float* std, const float* pre_hm,
                                       void* out, int32_t H, int32_t W, void* stream) {
  return pack_stem_frames_dev<false>(cur, prev, frames_dev, B, buf_bytes, mean, std, pre_hm, out, H, W, stream);
}

extern "C" int ct_pack_stem_frames_flip_dev(const uint8_t* cur, const uint8_t* prev, const ct_frame* frames_dev,
                                            int32_t B, int64_t buf_bytes, const float* mean, const float* std,
                                            const float* pre_hm, void* out, int32_t H, int32_t W, void* stream) {
  return pack_stem_frames_dev<true>(cur, prev, frames_dev, B, buf_bytes, mean, std, pre_hm, out, H, W, stream);
}

extern "C" int ct_warp_frames_normalize(const uint8_t* src, const ct_frame* frames_dev, int32_t B, int64_t buf_bytes,
                                        const float* mean, const float* std, float* dst, int32_t out_h, int32_t out_w,
                                        void* stream) {
  CT_REQUIRE(src && frames_dev && mean && std && dst, "null pointer");
  CT_REQUIRE(B > 0 && B <= 65535 && out_h > 0 && out_w > 0, "bad shape");
  CT_REQUIRE(buf_bytes >= 0, "buf_bytes < 0");
  // the same total as ct_warp_affine_normalize's grid-stride launch, split over the B streams
  const size_t plane = (size_t)out_h * out_w;
  const size_t cap = ((size_t)device_sm_count() * 16 + B - 1) / B;
  const size_t nx = (plane + 255) / 256 < cap ? (plane + 255) / 256 : cap;
  const DeviceFrames fs = {frames_dev, (long long)buf_bytes};
  warp_frames_norm_kernel<<<dim3((unsigned)nx, (unsigned)B), 256, 0, (cudaStream_t)stream>>>(
      src, fs, dst, out_h, out_w, make_float3(mean[0], mean[1], mean[2]), make_float3(std[0], std[1], std[2]));
  return after_launch();
}

// What ct_crop_boxes and ct_crop_boxes_tensor both refuse (the uint8 out is ct_crop_boxes' alone).
static int crop_desc_ok(const ct_crop_desc* d, const int32_t* streams, int32_t n, int32_t n_streams, bool u8_out) {
  CT_REQUIRE(d && d->buf && d->frames && d->rows && d->counts && (d->out || !u8_out) && d->out_counts, "null pointer");
  CT_REQUIRE(n > 0 && n <= 65535 && n_streams > 0, "bad batch (0 < n <= 65535, n_streams > 0)");
  CT_REQUIRE(d->K > 0 && d->K <= 65535 && d->out_h > 0 && d->out_w > 0, "bad shape (0 < K <= 65535, out_h, out_w > 0)");
  CT_REQUIRE(d->rows_per_stream > 0 && d->counts_stride > 0 && d->buf_bytes >= 0,
             "bad table (rows_per_stream > 0, counts_stride > 0, buf_bytes >= 0)");
  CT_REQUIRE(d->row_floats >= CT_TRK_BBOX + 4 && d->active_col >= -1 && d->active_col < d->row_floats,
             "row width does not contain the bbox or active column");
  CT_REQUIRE(streams || n <= n_streams, "without a stream map every image needs a stream (n <= n_streams)");
  const size_t total = (size_t)d->out_h * d->out_w;
  const size_t per_cta = (size_t)CROP_THREADS * CROP_PIX;
  CT_REQUIRE((total + per_cta - 1) / per_cta <= 0x7fffffffu, "crop too large");
  return CT_OK;
}

static dim3 crop_grid(const ct_crop_desc* d, int32_t n) {
  const size_t total = (size_t)d->out_h * d->out_w;
  const size_t per_cta = (size_t)CROP_THREADS * CROP_PIX;
  return dim3((unsigned)((total + per_cta - 1) / per_cta), (unsigned)d->K, (unsigned)n);
}

extern "C" int ct_crop_boxes(const ct_crop_desc* d, const int32_t* streams, int32_t n, int32_t n_streams,
                             void* stream) {
  if (const int e = crop_desc_ok(d, streams, n, n_streams, true)) return e;
  CropArgs a = {};
  a.d = *d;
  a.streams = streams;
  a.n_streams = n_streams;
  crop_boxes_kernel<CROP_U8><<<crop_grid(d, n), CROP_THREADS, 0, (cudaStream_t)stream>>>(a);
  return after_launch();
}

extern "C" int ct_crop_boxes_tensor(const ct_crop_desc* d, const ct_crop_tensor* t, const int32_t* streams, int32_t n,
                                    int32_t n_streams, void* stream) {
  if (const int e = crop_desc_ok(d, streams, n, n_streams, false)) return e;
  CT_REQUIRE(t && t->out && t->out_offsets, "null pointer");
  CT_REQUIRE(t->type == CT_CROP_F32 || t->type == CT_CROP_F16 || t->type == CT_CROP_BF16, "unknown element type");
  CT_REQUIRE(t->order == CT_CROP_RGB || t->order == CT_CROP_BGR, "unknown channel order");
  for (int c = 0; c < 3; ++c)
    CT_REQUIRE(isfinite(t->mean[c]) && isfinite(t->std[c]) && t->std[c] != 0.f, "mean and std must be finite, std != 0");
  const int64_t rows = (int64_t)n * d->K;
  CT_REQUIRE(rows <= 0x7fffffff, "n * K above 2^31 - 1 (int32 offsets)");
  CT_REQUIRE(t->rows_cap >= rows, "rows_cap < n * K");
  CT_REQUIRE(((uintptr_t)t->out & (t->type == CT_CROP_F32 ? 3 : 1)) == 0, "out not aligned to its element size");
  CropArgs a = {};
  a.d = *d;
  a.streams = streams;
  a.n_streams = n_streams;
  a.t = *t;
  crop_offsets_kernel<<<1, CROP_OFF_THREADS, 0, (cudaStream_t)stream>>>(a, n);
  if (const int e = after_launch()) return e;
  const dim3 grid = crop_grid(d, n);
  if (t->type == CT_CROP_F32) crop_boxes_kernel<CT_CROP_F32><<<grid, CROP_THREADS, 0, (cudaStream_t)stream>>>(a);
  else if (t->type == CT_CROP_F16) crop_boxes_kernel<CT_CROP_F16><<<grid, CROP_THREADS, 0, (cudaStream_t)stream>>>(a);
  else crop_boxes_kernel<CT_CROP_BF16><<<grid, CROP_THREADS, 0, (cudaStream_t)stream>>>(a);
  return after_launch();
}

extern "C" int ct_stage_frames(const ct_frame_src* srcs, const ct_frame* dst, int32_t n, uint8_t* buf,
                               int64_t buf_bytes, void* stream) {
  CT_REQUIRE(srcs && dst && buf, "null pointer");
  CT_REQUIRE(n > 0, "n <= 0");
  CT_REQUIRE(buf_bytes >= 0, "buf_bytes < 0");
  // everything is on the host: check every stream before the first launch
  for (int32_t i = 0; i < n; ++i) {
    const ct_frame_src& s = srcs[i];
    const ct_frame& f = dst[i];
    CT_REQUIRE(s.layout >= CT_SRC_BGR && s.layout <= CT_SRC_I420, "unknown source layout");
    const bool yuv = s.layout == CT_SRC_NV12 || s.layout == CT_SRC_I420;
    const int32_t fmt = s.layout == CT_SRC_NV12 ? CT_FRAME_NV12 : (s.layout == CT_SRC_I420 ? CT_FRAME_I420 : CT_FRAME_BGR);
    CT_REQUIRE(f.format == fmt, "source layout and destination format differ (BGR / RGB / RGB_PLANAR -> BGR, NV12 -> "
                                "NV12, I420 -> I420)");
    CT_REQUIRE(f.h > 0 && f.w > 0 && f.offset >= 0, "bad destination frame (h > 0, w > 0, offset >= 0)");
    CT_REQUIRE(f.h < (1 << 29) && f.w < (1 << 28), "frame too large");
    CT_REQUIRE(!yuv || ((f.h | f.w) & 1) == 0, "4:2:0 frames have an even height and width");
    const int planes = s.layout == CT_SRC_NV12 ? 2 : ((s.layout == CT_SRC_I420 || s.layout == CT_SRC_RGB_PLANAR) ? 3 : 1);
    const int64_t row[3] = {yuv || s.layout == CT_SRC_RGB_PLANAR ? f.w : 3LL * f.w,
                            s.layout == CT_SRC_I420 ? f.w / 2 : f.w, s.layout == CT_SRC_I420 ? f.w / 2 : f.w};
    for (int p = 0; p < planes; ++p) {
      CT_REQUIRE(s.plane[p] != nullptr, "null source plane");
      CT_REQUIRE(s.pitch[p] >= row[p], "source pitch shorter than a row");
    }
    const int64_t rows = yuv ? 3LL * (f.h / 2) : f.h, row_bytes = yuv ? f.w : 3LL * f.w;
    CT_REQUIRE(f.step >= row_bytes, "destination step shorter than a row");
    CT_REQUIRE(f.offset <= buf_bytes && (rows - 1) * f.step + row_bytes <= buf_bytes - f.offset,
               "destination extends past buf_bytes");
  }
  for (int32_t i0 = 0; i0 < n; i0 += CT_FRAMES_PER_LAUNCH) {
    const int m = n - i0 < CT_FRAMES_PER_LAUNCH ? n - i0 : CT_FRAMES_PER_LAUNCH;
    StageArgs a = {};
    int64_t most = 0;
    for (int i = 0; i < m; ++i) {
      const ct_frame_src& s = srcs[i0 + i];
      const ct_frame& f = dst[i0 + i];
      StageFrame& g = a.f[i];
      for (int p = 0; p < 3; ++p) {
        g.src[p] = (const unsigned char*)s.plane[p];
        g.pitch[p] = s.pitch[p];
      }
      g.offset = f.offset;
      g.h = f.h, g.w = f.w, g.step = f.step, g.layout = s.layout;
      const int64_t rows = s.layout == CT_SRC_NV12 ? f.h + f.h / 2 : (s.layout == CT_SRC_I420 ? 2LL * f.h : f.h);
      most = rows > most ? rows : most;
    }
    const dim3 grid((unsigned)((most + STAGE_WARPS - 1) / STAGE_WARPS), (unsigned)m);
    stage_frames_kernel<<<grid, STAGE_THREADS, 0, (cudaStream_t)stream>>>(a, buf);
    const int rc = after_launch();
    if (rc != CT_OK) return rc;
  }
  return CT_OK;
}
