/* ctb200.h -- C ABI of libctb200.so: the H100 (sm_90a) implementation of CenterTrack's
 * per-frame inference hot path.  Plain C: raw device pointers, sizes, a cudaStream_t passed
 * as void*; every entry point returns 0 on success or a negative ct_status and never throws.
 * No ownership transfer: the caller (the Python shims in centertrack_b200/, which allocate
 * through torch) owns every buffer.  Thread-compatible: no global mutable state other than
 * the per-thread last-error string.
 *
 * Reference interfaces each entry point replaces (paths relative to the reference's src/lib):
 *   ct_conv_forward   nn.Conv2d+BatchNorm2d(+residual)+ReLU chains of DLA-34: dla.py:38-66
 *                     (BasicBlock), 154-172 (Root), 293-303 (_make_conv_level), 212-218
 *                     (Tree.project); head convs base_model.py:27-38; and, with
 *                     mode=CT_A_DCN, the absent DCNv2 extension's DCN.forward that
 *                     dla.py:513,516 calls (modulated deformable conv v2, 3x3/s1/p1/dg1).
 *   ct_stem_forward   DLA.forward's three 7x7 stems, dla.py:238-242,256-267,305-311.
 *   ct_maxpool2       nn.MaxPool2d(2,2) = Tree.downsample, dla.py:207.
 *   ct_upsample_add   IDAUp's depthwise ConvTranspose2d + skip add, dla.py:529-531,543-545.
 *   ct_decode         Detector.process's decode half: _nms + _topk + _tranpose_and_gather_feat
 *                     + generic_decode, utils.py:16-26,52-87 and decode.py:83-182
 *                     (+ _update_kps_with_hm decode.py:11-81 for the pose heads).
 *   ct_render_pre_hm  Detector._get_additional_inputs's gaussian splat, detector.py:254-290.
 *   ct_track_step     generic_post_process's affine (utils/post_process.py:21-91) + Tracker.step's greedy association
 *                     (utils/tracker.py:28-138) + the (centre, radius) boxes of _get_additional_inputs for the next
 *                     frame, per stream, on the device;  ct_render_tracks splats those boxes (image.py:128-154).
 *                     ct_track_step_assoc adds --hungarian and --public_det association (tracker.py:52-72,83-103);
 *                     ct_track_step_payload adds the pose / 3D / velocity / attribute fields (post_process.py:55-89).
 *                     ct_track_start: reset_tracking + Tracker.init_track(pre_dets) on some streams alone
 *                     (detector.py:97-103, utils/tracker.py:11-22).
 *   ct_flip_merge     Detector._flip_output, detector.py:311-332 (flip_tensor / flip_lr / flip_lr_off, model/utils.py:28-50);
 *                     ct_flip_merge_heads merges every head of B pairs at once, ct_mirror_x mirrors the --flip_test
 *                     batch's second half (detector.py:225-226,285-286).
 *   ct_warp_affine_normalize   Detector.pre_process's cv2.warpAffine + normalise + HWC->CHW, detector.py:207-226.
 *   ct_pack_stem_frames        the same for B ragged uint8 frames and their previous frames, written as the packed
 *                     input of the tensor-core stem (no fp32 image in between); ct_pack_stem_frames_flip also writes
 *                     each stream's mirror image for --flip_test.
 */
#ifndef CTB200_H_
#define CTB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CTB200_ABI_VERSION 1

typedef enum {
  CT_OK = 0,
  CT_ERR_INVALID = -1,     /* bad argument / unsupported shape */
  CT_ERR_CUDA = -2,        /* a CUDA runtime call failed (see ct_last_error) */
  CT_ERR_UNSUPPORTED = -3  /* valid request this build cannot serve */
} ct_status;

typedef enum { CT_F32 = 0, CT_BF16 = 1 } ct_dtype;

/* How the A operand (rows = output pixels, K = taps x C_in) of the implicit GEMM is formed. */
typedef enum {
  CT_A_CONV = 0,  /* plain KxK window, stride/pad */
  CT_A_DCN = 1,   /* 3x3 s1 p1 modulated-deformable bilinear sampling driven by `om` */
  CT_A_DCN_WIN = 2 /* the same operator on the bf16 wgmma engine with the input neighbourhood of each 8x16-pixel
                      output patch staged in shared memory by TMA (samples displaced by more than the margin fall
                      back to global memory).  Needs C_in % 64 == 0 and weights packed 64-channel-chunk-major:
                      ct_pack_weights(engine, w', C_out, 64, 3 * C_in / 64, 3, ...) with
                      w'[o][c][chunk * 3 + ky][kx] = w[o][chunk * 64 + c][ky][kx] */
} ct_a_mode;

/* Epilogue / output format. */
typedef enum {
  CT_OUT_NHWC = 0,       /* out[p*ld_out + o], activation dtype */
  CT_OUT_NHWC_F32 = 1,   /* fp32 NHWC (DCN offset/mask map; sigmoid on channels >= sig_from) */
  CT_OUT_NCHW_F32 = 2,   /* fp32 [B,C_out,H,W] planes (head outputs, reference layout) */
  CT_OUT_NHWC_S2D = 3    /* CT_OUT_NHWC written space-to-depth: pixel (y, x) lands at pixel (y/2, x/2), channels
                            [((y&1)*2 + (x&1)) * ld_out, +C_out) of a [B, OH/2, OW/2, 4*ld_out] tensor -- the input
                            layout of a stride-2 3x3 consumer run as a stride-1 2x2 convolution over 4*C channels
                            (DLA stem -> level0 -> level1).  Halo engine only; OH, OW even; no residual. */
} ct_out_mode;

typedef enum {           /* per-launch transform applied to the fp32 NCHW head outputs */
  CT_HEAD_NONE = 0,
  CT_HEAD_SIGMOID = 1,   /* hm, hm_hp: detector.py:301-304 */
  CT_HEAD_DEPTH = 2      /* dep = 1/(sigmoid(x)+1e-6)-1, times depth_scale: detector.py:305-307 */
} ct_head_act;

typedef enum {
  CT_ENGINE_SIMT = 0,          /* fp32 FFMA implicit GEMM (reference accuracy; fp32 or bf16 activations) */
  CT_ENGINE_TCGEN05 = 1,       /* wgmma implicit GEMM, A gathered per tap (any stride, DCN) */
  CT_ENGINE_TCGEN05_HALO = 2,  /* wgmma, TMA-loaded halo tile, taps by descriptor shift: stride-1 'same'
                                  convs with C_in in {8,16,32,48,64,128,192,256} whose weights fit in smem */
  CT_ENGINE_TCGEN05_X3 = 3     /* the gather engine on fp32 activations (dtype CT_F32) with bf16 hi/lo split operands:
                                  D += A_hi B_hi + A_hi B_lo + A_lo B_hi, fp32 accumulate -- ~1e-5 per layer, the
                                  tensor-core path that meets the reference's fp32 results to 1e-3 end to end */
} ct_engine;

/* One output head of a fused head launch (ct_conv_desc.n_heads > 0): the head's 1x1 convolution over its mid_c
 * channels of the shared 3x3 layer, + bias, head_act, written as an fp32 NCHW map. */
#define CT_MAX_FUSED_HEADS 12
typedef struct {
  const void* w;         /* 1x1 weights [C_out, mid_c] packed by ct_pack_weights(CT_ENGINE_TCGEN05_HALO, .., n_tile) */
  const float* bias;     /* [C_out] */
  float* out;            /* fp32 [B, C_out, OH, OW] */
  int32_t C_out;
  int32_t n_tile;        /* multiple of 16, C_out <= n_tile <= 80 */
  int32_t head_act;      /* ct_head_act */
  int32_t reserved;
} ct_head;

/* One convolution-like layer.  Activations are NHWC with an explicit pixel stride (ld, in
 * elements) so that a producer can write straight into a channel slice of a concat buffer
 * (DLA Root nodes, dla.py:167) and a consumer can read a slice back. */
typedef struct {
  int32_t engine;        /* ct_engine */
  int32_t dtype;         /* ct_dtype of activations in/out (CT_ENGINE_TCGEN05 requires CT_BF16) */
  int32_t a_mode;        /* ct_a_mode */
  int32_t B, H, W;       /* input batch / spatial size */
  int32_t C_in, ld_in;   /* input channels used, input pixel stride */
  int32_t C_out;         /* real output channels */
  int32_t KH, KW, stride, pad;
  int32_t OH, OW;        /* output spatial size */
  int32_t ld_out;        /* output pixel stride (CT_OUT_NHWC*; CT_OUT_NHWC_S2D: stride of one of the four sub-pixels) */
  int32_t out_mode;      /* ct_out_mode */
  int32_t relu;          /* 1: ReLU after shift (+residual) */
  int32_t ld_res;        /* residual pixel stride (residual may be NULL) */
  int32_t head_act;      /* ct_head_act (CT_OUT_NCHW_F32 only) */
  int32_t sig_from;      /* CT_OUT_NHWC_F32: sigmoid applied to channels >= sig_from (DCN mask) */
  float   depth_scale;
  int32_t ld_om;         /* CT_A_DCN: pixel stride of `om` (fp32 NHWC, >= 27) */
  int32_t n_tile;        /* wgmma engines: output-channel tile (multiple of 16, <= 256; required) */
  int32_t epilogue_sum3; /* HALO engine, C_out == 48: out16 = sum over present groups g (bit g set) of
                            relu(acc[16g..16g+15] + shift) -- the three DLA stems (dla.py:307-311) */
  int32_t pad_w1;        /* 0: horizontal padding = pad; else horizontal padding + 1 (the (k,1) / (1,k) convs of
                            GlobalConv, dla.py:477-503; SIMT and gather engines) */
  const void* x;         /* input activations */
  const void* w;         /* packed weights: see ct_pack_weights */
  const float* shift;    /* [C_out] folded BN shift / conv bias (may be NULL) */
  const void* residual;  /* [P_out, ld_res] same dtype as activations, or NULL */
  const float* om;       /* CT_A_DCN: offsets (ch 0..17, 2k=dy 2k+1=dx) + sigmoid'd mask (18..26) */
  void* out;
  /* Fused output heads (HALO engine; 0 = an ordinary layer): the layer is the heads' shared 3x3 convolution
   * C_in = 64 -> C_out = n_heads * mid_c (mid_c = 64 or 256, n_tile = 64 or 128 = the mid channels per pass, relu,
   * shift = its bias), and each head's 1x1 runs on its mid_c channels in the same launch: the 3x3 result never leaves
   * the chip.  out_mode = CT_OUT_NCHW_F32, `out` is unused, the head outputs are heads[i].out. */
  int32_t n_heads;
  const ct_head* heads;  /* [n_heads] */
} ct_conv_desc;

/* Size in bytes of the packed weight blob ct_pack_weights produces for this engine/shape. */
int64_t ct_packed_weight_bytes(int32_t engine, int32_t C_out, int32_t C_in, int32_t KH, int32_t KW,
                               int32_t n_tile);
/* Host-side packing.  w_oihw: fp32 [C_out, C_in, KH, KW] (already BN-scale-folded).
 * SIMT engine : fp32 [KH*KW*C_in (k = tap*C_in + c)][C_out padded to 64].
 * wgmma       : bf16 tiles [n_tiles][k_slices][n_tile rows x 64 k] in the 128B-swizzled
 *               shared-memory image the MMA descriptor expects (one bulk copy per tile).
 * wgmma x3    : the same with two tiles per K slice: [hi = bf16(w)][lo = bf16(w - hi)].
 * wgmma halo  : bf16 [n_tiles][K=16 blocks][2 K-cores][n_tile/8][8 rows][8] (un-swizzled K-major core
 *               matrices); block = (tap, 16 channels), or (ky, tap pair) when C_in == 8. */
int ct_pack_weights(int32_t engine, const float* w_oihw, int32_t C_out, int32_t C_in, int32_t KH,
                    int32_t KW, int32_t n_tile, void* dst);

int ct_conv_forward(const ct_conv_desc* d, void* stream);

/* Launch configuration ct_conv_forward picks for a descriptor (ct_conv_config). */
struct ct_conv_config {
  int32_t smem_bytes;    /* dynamic shared memory per CTA (0: SIMT engine) */
  int32_t stages;        /* pipeline stages: halo tiles (HALO) or K slices (gather engines) in flight */
  int32_t tile_w, tile_h;/* output pixels of one work item: 8 x 16 or 32 x 4 (HALO); 16 x 8 patches or 128 x 1
                            consecutive pixels (gather engines) */
  int32_t ctas_per_sm;   /* HALO: CTAs per SM the persistent grid is sized for; 0 for the other engines */
  int32_t overlap;       /* HALO: 1 = the one-CTA-per-SM flavour whose two warpgroups take turns on the tensor cores */
};
/* The configuration step of ct_conv_forward alone: validates the descriptor's shape and fills `out`, with no CUDA
 * call.  Returns the status and ct_last_error() message ct_conv_forward would return for this shape
 * (CT_ERR_UNSUPPORTED: the tile does not fit in shared memory).  Of the pointer fields of `d` only whether residual
 * and shift are NULL is read (a layer without residual / shift), and the head table of a fused head launch (its
 * C_out / n_tile); the others may be NULL.  Fused heads: `stages` counts the weight-slice ring. */
int ct_conv_config(const ct_conv_desc* d, struct ct_conv_config* out);

/* Three 7x7 stems on reference-layout inputs (fp32 NCHW):
 *   out = relu(bn(conv7(img))) + relu(bn(conv7(pre_img))) + relu(bn(conv7(pre_hm)))
 * w: fp32 [49 taps][7 in-ch (img0..2, pre0..2, hm)][16] BN-scale-folded; shift: [3][16].
 * pre_img / pre_hm may be NULL (dla.py:308-311).  out: NHWC [B,H,W,16] of `dtype`. */
int ct_stem_forward(const float* img, const float* pre_img, const float* pre_hm, const float* w,
                    const float* shift, void* out, int32_t dtype, int32_t B, int32_t H, int32_t W,
                    int32_t ld_out, void* stream);

/* (img, pre_img, pre_hm) fp32 NCHW -> bf16 NHWC [B,H,W,8] = (img0..2, pre0..2, hm, 0): the input of the
 * tensor-core stem (CT_ENGINE_TCGEN05_HALO, 7x7, C_in = 8, epilogue_sum3).  NULL inputs give zeros. */
int ct_pack_stem_input(const float* img, const float* pre_img, const float* pre_hm, void* out, int32_t B,
                       int32_t H, int32_t W, void* stream);

/* the same packing in fp32 (NHWC [B,H,W,8] floats): stem input of CT_ENGINE_TCGEN05_X3 */
int ct_pack_stem_input_f32(const float* img, const float* pre_img, const float* pre_hm, float* out, int32_t B,
                           int32_t H, int32_t W, void* stream);

int ct_maxpool2(const void* x, void* out, int32_t dtype, int32_t B, int32_t H, int32_t W, int32_t C,
                int32_t ld_in, int32_t ld_out, void* stream);

/* the same pooling of a tensor stored space-to-depth (CT_OUT_NHWC_S2D): x [B,H2,W2,(sy,sx,C)] -> out [B,H2,W2,C],
 * out[p][c] = max over the four C-channel groups of pixel p */
int ct_maxpool2_s2d(const void* x, void* out, int32_t dtype, int32_t B, int32_t H2, int32_t W2, int32_t C,
                    int32_t ld_in, int32_t ld_out, void* stream);

/* out[b,oy,ox,c] = skip[...] + sum_{ky,kx} x[b,(oy+pad-ky)/f,(ox+pad-kx)/f,c] * w[ky,kx,c]
 * (depthwise ConvTranspose2d, kernel 2f, stride f, pad f/2; w fp32 channel-last [2f][2f][C]). */
int ct_upsample_add(const void* x, const void* skip, const float* w, void* out, int32_t dtype,
                    int32_t B, int32_t H, int32_t W, int32_t C, int32_t f, int32_t ld_in,
                    int32_t ld_skip, int32_t ld_out, void* stream);

/* ---- decode ------------------------------------------------------------------------- */
#define CT_DECODE_MAX_HEADS 12
typedef enum {          /* role of a gathered regression map in generic_decode */
  CT_ROLE_RAW = 0,      /* copied as-is (tracking, dep, rot, dim, amodel_offset, ...) */
  CT_ROLE_REG = 1,      /* center offset: xs = xs0 + reg_x (decode.py:103-108) */
  CT_ROLE_WH = 2,       /* clamped >= 0, makes bboxes (decode.py:113-129) */
  CT_ROLE_LTRB = 3,     /* bboxes = ct0 + ltrb (decode.py:132-139) */
  CT_ROLE_LTRB_AMODAL = 4, /* bboxes_amodal, overrides bboxes (decode.py:150-159) */
  CT_ROLE_HPS = 5       /* keypoint offsets: += xs0/ys0 (decode.py:161-166) */
} ct_head_role;

typedef struct {
  const float* map;     /* fp32 [B, channels, H, W] */
  int32_t channels;
  int32_t role;         /* ct_head_role */
  int32_t rec_offset;   /* float offset inside a record where the raw gathered row is written */
} ct_decode_head;

typedef struct {
  int32_t B, C, H, W, K;
  const float* hm;          /* post-sigmoid fp32 [B,C,H,W] */
  int32_t n_heads;
  ct_decode_head heads[CT_DECODE_MAX_HEADS];
  /* pose refinement (decode.py:11-81); hm_hp == NULL disables */
  const float* hm_hp;       /* post-sigmoid [B,J,H,W] */
  const float* hp_offset;   /* [B,2,H,W] or NULL (then `reg` head map is used if present, else +0.5) */
  int32_t J;
  int32_t rec_hps;          /* float offset of the 2J refined keypoints, -1 if none */
  int32_t rec_kps_score;    /* float offset of kps_score, -1 if none */
  /* record layout: [score, cls, xs0, ys0, bbox l,t,r,b, ind (int32 bits), ... heads ...] */
  int32_t rec_floats;       /* floats per record (F) */
  int32_t has_bbox;
  float*  records;          /* out [B, K, F] */
  /* workspace: ct_decode_workspace_bytes(...) bytes, 256B aligned; contents need no init
   * except that the first 4*B bytes (per-batch arrival counters) are zeroed by the caller
   * once; the kernel resets them. */
  void* workspace;
} ct_decode_desc;

#define CT_REC_SCORE 0
#define CT_REC_CLS 1
#define CT_REC_XS 2
#define CT_REC_YS 3
#define CT_REC_BBOX 4
#define CT_REC_IND 8
#define CT_REC_HEADS 9

int64_t ct_decode_workspace_bytes(int32_t B, int32_t C, int32_t J, int32_t K);
int ct_decode(const ct_decode_desc* d, void* stream);

/* Gaussian splat of the previous frame's tracks into pre_hm (fp32 [B,1,H,W], zeroed here).
 * boxes: fp32 [n,5] rows (b, cx_int, cy_int, radius, unused) already in INPUT-resolution
 * pixel units -- the affine + gaussian_radius arithmetic stays on the host
 * (detector.py:264-276); the np.maximum splat of image.py:138-154 runs on the device. */
int ct_render_pre_hm(const float* boxes, int32_t n, float* pre_hm, int32_t B, int32_t H, int32_t W,
                     void* stream);

/* ---- per-stream state on the device (SURVEY 8f) ------------------------------------------ */
/* One track / result row: the fields Tracker.step reads and writes (utils/tracker.py), image coordinates. */
#define CT_TRK_SCORE 0
#define CT_TRK_CLASS 1      /* clses + 1 (post_process.py:47) */
#define CT_TRK_CT 2         /* ct x, y */
#define CT_TRK_TRACKING 4   /* tracking dx, dy (already in image coordinates) */
#define CT_TRK_BBOX 6       /* x0, y0, x1, y1 */
#define CT_TRK_ID 10        /* tracking_id (exact in fp32 below 2^24) */
#define CT_TRK_AGE 11
#define CT_TRK_ACTIVE 12
#define CT_TRK_FLOATS 13

typedef struct {
  int32_t B, K, F;            /* decode records [B,K,F] (ct_decode), sorted by score */
  int32_t rec_tracking;       /* float offset of the `tracking` head inside a record, -1 if absent */
  int32_t max_tracks;         /* T: rows of the per-stream track table (>= K; tracks beyond T are dropped) */
  float out_thresh;           /* detections with score > out_thresh survive (detector.py:371-377) */
  float new_thresh;           /* unmatched detections with score > new_thresh start a track (tracker.py:108-113) */
  float pre_thresh;           /* tracks with score >= pre_thresh and active != 0 are splatted (detector.py:262-263) */
  int32_t max_age;            /* unmatched tracks coast while age < max_age (tracker.py:115-126) */
  int32_t inp_h, inp_w;       /* network input size = pre_hm size */
  const float* records;
  const float* trans_out_inv; /* [B,6] fp32: output grid -> image, get_affine_transform(c,s,0,(w,h),inv=1).astype(f32) */
  const double* trans_input;  /* [B,6] fp64: image -> network input (meta['trans_input']); needed when boxes != NULL */
  float* tracks;              /* in/out [B,T,CT_TRK_FLOATS]: the stream's tracks == the results of this step */
  int32_t* counts;            /* in/out [B,2]: number of tracks, id_count */
  float* boxes;               /* out [B,T,5] rows (b, cx, cy, radius, 0) for ct_render_tracks, radius < 0 = skip; or NULL */
} ct_track_desc;

/* Association mode of ct_track_step_assoc (tracker.py:52-72,83-103).  All zero = ct_track_step. */
typedef struct {
  int32_t hungarian;          /* 1: --hungarian, scipy.optimize.linear_sum_assignment's assignment (same tie-breaking) */
  int32_t public_det;         /* 1: --public_det, tracks are born only where a public detection claims a detection */
  int32_t max_public;         /* P: row stride of public_ct (> 0 when public_det) */
  const float* public_ct;     /* [B,P,2] fp32 public detection centres, image coordinates; needed when public_det */
  const int32_t* public_n;    /* [B] public detections of each stream (clamped to [0, P] on the device) */
  int32_t* steps;             /* out [B] Dijkstra search steps of this frame's Hungarian solve (0 if none), or NULL */
} ct_track_assoc;

int64_t ct_track_smem_bytes(int32_t K, int32_t max_tracks);
int ct_track_step(const ct_track_desc* d, void* stream);
/* Shared memory of ct_track_step_assoc with hungarian or public_det set (the solver's scratch comes on top). */
int64_t ct_track_assoc_smem_bytes(int32_t K, int32_t max_tracks);
/* ct_track_step with the association mode `a`: same kernel, same phases; the greedy, private-birth path is
 * ct_track_step's.  Unmatched detections / tracks are born / coast in the reference's order (naturally unmatched
 * ascending, then those of rejected Hungarian pairs in pair order); public births come in public-detection order. */
int ct_track_step_assoc(const ct_track_desc* d, const ct_track_assoc* a, void* stream);

/* Task fields of generic_post_process (post_process.py:55-89) kept beside the track table: payload row r belongs to
 * track row r, written by the same launch in the same order; coasting tracks keep theirs unchanged.  A row holds, in
 * this order and each only when its record offset is >= 0:
 *   hps [hps_floats]        keypoints through the output affine (rec_hps: the refined keypoints when decode refined them)
 *   dep [1], dim [3]        copied
 *   alpha [1]               get_alpha(rot)                                          (rec_rot)
 *   loc [3], rot_y [1]      ddd2locrot(amodal centre, alpha, dim, dep, calib[b])    (rec_rot, rec_dep and rec_dim)
 *   velocity [velocity_floats], nuscenes_att [att_floats]   copied
 * With rot, dep and dim all present the track's CT_TRK_CT is the reference's amodal centre (the output-grid box centre
 * + amodel_offset through the affine, or the image box centre without rec_amodel_offset), and association runs on it;
 * CT_TRK_TRACKING stays relative to the heat-map peak. */
typedef struct {
  int32_t width;              /* Wp: floats per payload row = the sum of the enabled fields' widths */
  float* payload;             /* in/out [B,T,Wp] */
  int32_t rec_hps, hps_floats;
  int32_t rec_dep, rec_dim, rec_rot, rec_amodel_offset;
  int32_t rec_velocity, velocity_floats;
  int32_t rec_nuscenes_att, att_floats;
  const float* calib;         /* [B,3,4] fp32 camera matrices; needed when rot, dep and dim are all present */
} ct_track_payload;

/* Shared memory of ct_track_step_payload: the table (with the association scratch when assoc != 0) + T payload rows. */
int64_t ct_track_payload_smem_bytes(int32_t K, int32_t max_tracks, int32_t width, int32_t assoc);
/* ct_track_step_assoc that also writes the payload table; p == NULL is ct_track_step_assoc. */
int ct_track_step_payload(const ct_track_desc* d, const ct_track_assoc* a, const ct_track_payload* p, void* stream);
/* Start a new video on some streams (Detector.reset_tracking + Tracker.init_track on those streams alone): for each of
 * the n_starts entries of `starts` (device int32 [n_starts][2] = (stream, seed rows n), distinct streams in [0, B)), the
 * stream's T track rows, its counts and (p != NULL) its payload rows are zeroed, its n seed rows are written (fp32
 * [n][CT_TRK_FLOATS] in track-table format, already filtered and numbered: ids 1..n), counts = (n, n), and its T render
 * boxes are computed from them as ct_track_step computes them.  `seeds` (device) holds the rows of entry 0, then entry 1,
 * ...; it may be NULL when no entry has seeds.  n is clamped to [0, T] and entries with a stream outside [0, B) are
 * skipped on the device.  Every other stream is left untouched.  One CTA per entry; n_starts == 0 launches nothing.
 * Only d->B, max_tracks, pre_thresh, inp_h, inp_w, trans_input, tracks, counts and boxes are read. */
int ct_track_start(const ct_track_desc* d, const ct_track_payload* p, const int32_t* starts, int32_t n_starts,
                   const float* seeds, void* stream);
/* pre_hm (fp32 [B,1,H,W], zeroed here) <- max-splat of boxes [n,5] (rows with radius < 0 skipped); n is the grid size,
 * so the launch shape does not depend on the data (CUDA-graph capturable). */
int ct_render_tracks(const float* boxes, int32_t n, float* pre_hm, int32_t B, int32_t H, int32_t W, void* stream);

/* out[c,y,x] = (in2[0,c,y,x] + sign[c] * in2[1,perm[c],y,W-1-x]) / 2;  in2 fp32 [2,C,H,W], out [1,C,H,W];
 * perm (int32 [C], device) / sign (fp32 [C], device) may be NULL (identity / +1). */
int ct_flip_merge(const float* in2, float* out, int32_t C, int32_t H, int32_t W, const int32_t* perm,
                  const float* sign, void* stream);

/* One averaged head of a --flip_test batch of B (frame, mirrored frame) pairs: frames [0, B), mirrors [B, 2B). */
typedef struct {
  const float* in;            /* fp32 [2B,C,H,W] (device) */
  float* out;                 /* fp32 [B,C,H,W] (device) */
  int32_t C;
  int32_t reserved;
  const int32_t* perm;        /* int32 [C] (device) or NULL = identity */
  const float* sign;          /* fp32 [C] (device) or NULL = +1 */
} ct_flip_head;

/* Heads per ct_flip_merge_heads launch (the descriptors travel in the kernel parameters). */
#define CT_FLIP_MAX_HEADS 12

/* ct_flip_merge of every head in `heads` (HOST array [n_heads], read during the call and passed to the kernel by
 * value, so a captured CUDA graph keeps it) and of all B pairs, in one launch:
 *   out[b,c,y,x] = (in[b,c,y,x] + sign[c] * in[B+b,perm[c],y,W-1-x]) / 2, with ct_flip_merge's rounding.
 * ct_flip_merge is the case n_heads = 1, B = 1. */
int ct_flip_merge_heads(const ct_flip_head* heads, int32_t n_heads, int32_t B, int32_t H, int32_t W, void* stream);

/* dst[i,c,y,x] = src[i,c,y,W-1-x] for fp32 [n,C,H,W] (device, non-overlapping): the mirrored half of a --flip_test
 * batch. */
int ct_mirror_x(const float* src, float* dst, int32_t n, int32_t C, int32_t H, int32_t W, void* stream);

/* dst fp32 [B,3,out_h,out_w] = ((warpAffine(src) / 255 - mean) / std), src uint8 [B,src_h,src_w,3] (row pitch src_step
 * bytes), minv fp64 [B,6] = the INVERTED 2x3 map (dst -> src) exactly as cv::warpAffine inverts it; mean/std host fp32[3].
 * Bilinear in cv2's fixed point (1/32 px, 15-bit weights), zero border. */
int ct_warp_affine_normalize(const uint8_t* src, int32_t B, int32_t src_h, int32_t src_w, int32_t src_step,
                             const double* minv, const float* mean, const float* std, float* dst, int32_t out_h,
                             int32_t out_w, void* stream);

/* One stream's frame inside a buffer of B ragged uint8 BGR frames (StreamRunner's frame slots). */
typedef struct {
  int64_t offset;             /* byte offset of the frame in the buffer (StreamRunner aligns it to 16 bytes) */
  int32_t h, w, step;         /* source rows, columns, row pitch in bytes (>= 3 w) */
  int32_t reserved;
  double  minv[6];            /* dst -> src map, inverted exactly as cv::warpAffine inverts it (see above) */
} ct_frame;

/* Streams per kernel launch of ct_pack_stem_frames (the descriptors travel in the kernel parameters). */
#define CT_FRAMES_PER_LAUNCH 48

/* out bf16 NHWC [B,H,W,8] = (norm(warp(cur_b)) x3, norm(warp(prev_b)) x3, pre_hm_b, 0): the tensor-core stem's input,
 * byte-identical to ct_warp_affine_normalize of each stream followed by ct_pack_stem_input.  cur / prev: device buffers
 * holding each stream's frame at frames[b].offset (the same descriptor is used for both); prev == NULL or
 * pre_hm == NULL (fp32 [B,1,H,W]) give zeros.  frames: HOST array [B], read during the call and passed to the kernels
 * by value (a captured CUDA graph keeps them); one launch per CT_FRAMES_PER_LAUNCH streams.  mean / std host fp32[3]. */
int ct_pack_stem_frames(const uint8_t* cur, const uint8_t* prev, const ct_frame* frames, int32_t B, const float* mean,
                        const float* std, const float* pre_hm, void* out, int32_t H, int32_t W, void* stream);
/* --flip_test: ct_pack_stem_frames into out [2B,H,W,8] whose image B+b is image b mirrored along W (out[B+b][y][W-1-x]
 * = out[b][y][x]), as if frame, previous frame and pre_hm had all been mirrored.  Same arguments; pre_hm stays [B,1,H,W]
 * (un-mirrored). */
int ct_pack_stem_frames_flip(const uint8_t* cur, const uint8_t* prev, const ct_frame* frames, int32_t B,
                             const float* mean, const float* std, const float* pre_hm, void* out, int32_t H, int32_t W,
                             void* stream);

/* ---- misc --------------------------------------------------------------------------- */
const char* ct_last_error(void);
int ct_abi_version(void);
/* Kernels launched by this library on the calling thread since the last reset. */
int64_t ct_launch_count(void);
void ct_reset_launch_count(void);
/* Debug: timeline trace of CTA 0 of the halo conv kernel into device_buf (>= 16 KB of uint64: 8 clock64()
 * stamps per work item, see csrc/conv_halo.cu); NULL switches it off (default). */
int ct_debug_trace(void* device_buf);
/* Debug: 4 uint32 of host-MAPPED memory; a stuck mbarrier wait in any kernel of the library (halo and gather
 * convolutions, decode) writes (site, item, block, warp) there before trapping.  NULL = off (default). */
int ct_debug_watch(void* mapped_host_buf);

#ifdef __cplusplus
}
#endif
#endif /* CTB200_H_ */
