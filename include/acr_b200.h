/* acr_b200.h -- C ABI of the H100-native (sm_90a) ACR hot path (libacr_b200.so).
 *
 * The reference (ZhengdiYu/Arbitrary-Hands-3D-Reconstruction) has no FFI of its own: its
 * boundary is a Python call surface (SURVEY.md section 8b).  Each entry point below names
 * the reference function(s) it replaces (path:line in /root/reference).  Conventions:
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless marked host;
 *   - `stream` is a cudaStream_t passed as void*; nothing synchronises, nothing allocates
 *     device memory (the caller owns all buffers and the plan arena);
 *   - return 0 on success, <0 on error; acr_b200_last_error() describes the last failure
 *     of the calling thread;
 *   - thread-compatible: concurrent calls must use different streams / plans.
 */
#ifndef ACR_B200_H_
#define ACR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ACR_B200_OK 0
#define ACR_B200_EINVAL (-1)
#define ACR_B200_ECUDA (-2)
#define ACR_B200_ENOTSUP (-3)

const char* acr_b200_last_error(void);
/* "acr_b200 <version> sm_90a" */
const char* acr_b200_version(void);

/* ------------------------------------------------------------------------------------------
 * MANO
 * ---------------------------------------------------------------------------------------- */
/* Number of floats in one packed MANO model and the packing itself (host side, once per
 * asset).  Replaces the buffer registration of ManoLayer.__init__ (mano/manolayer.py:59-102)
 * plus MANOWrapper's left-hand shapedirs x-flip (acr/mano_wrapper.py:35, `flip_x`).
 * Inputs are HOST row-major fp32 arrays: shapedirs (778,3,10), posedirs (778,3,135),
 * v_template (778,3), j_regressor (16,778), weights (778,16), hands_mean (45).          */
size_t acr_b200_mano_model_floats(void);
int acr_b200_mano_pack_model(const float* shapedirs, const float* posedirs, const float* v_template,
                             const float* j_regressor, const float* weights, const float* hands_mean,
                             int flip_x, float* packed_host);

/* Fused MANO forward + weak-perspective projection for n hands.
 * Replaces ManoLayer.forward (mano/manolayer.py:104-276: Rodrigues :423-434, pose/shape blend
 * :175-182, joint regression :178, kinematic chain :187-223, LBS :226-240, tips/reorder/centre
 * :241-261), MANOWrapper.forward's two-layer dispatch (acr/mano_wrapper.py:40-46) and
 * batch_orth_proj / convert_kp2d_from_input_to_orgimg (acr/utils.py:384-397).
 *   model_l/model_r : packed models (device); either may be NULL if that side never occurs
 *   poses (n,48) axis-angle [root|hand] WITHOUT the mean pose; betas (n,10)
 *   hand_type (n) int32 0=left 1=right, or NULL => every row uses `default_side`
 *   n_dev : optional device int32; rows >= *n_dev are skipped (lets a CUDA graph run with
 *           the worst-case n = n_max and no host sync).  NULL => all n_max rows.
 *   center_idx : joint (after reordering) subtracted from joints and vertices, -1 = none
 *   cam (n,3) [s,tx,ty] and offsets (n,10) optional (NULL => projection outputs skipped)
 * Outputs (any may be NULL): verts (n,778,3), joints (n,21,3), center (n,3),
 *   verts_camed (n,778,3), pj2d (n,21,2), pj2d_org (n,21,2).                              */
int acr_b200_mano_forward(const float* model_l, const float* model_r, const float* poses,
                          const float* betas, const int32_t* hand_type, int default_side,
                          const int32_t* n_dev, int n_max, int center_idx, const float* cam,
                          const float* offsets, float* verts, float* joints, float* center,
                          float* verts_camed, float* pj2d, float* pj2d_org, void* stream);

/* Same kernel, with the vertex all-gather FUSED into it (replaces the gather step of nn.DataParallel,
 * acr/main.py:61 / the separate ncclAllGather of SURVEY.md 8e).  Besides the local outputs, every vertex is
 * stored straight into the gather buffers of ALL ranks over NVLink: 16-byte `multimem.st.v4.f32` through the
 * NVLS multicast mapping (the NVSwitch replicates the store) or, when `multicast_base` is 0, one 16-byte peer
 * store per rank.  The 8 int32 row counts of the shard (`counts_src`, as written by acr_b200_parse) travel the
 * same way, so the exchange needs no other collective.
 *
 * Symmetric allocation (identical layout on every rank, e.g. torch symmetric memory / CUDA IPC / VMM):
 *     [ slot 0 | slot 1 | flags ]          slot = verts[world][rows][778][3] fp32 at 0,
 *                                                 counts[world][8] int32 at counts_offset
 *     flags = uint64[world] at flags_offset (from the allocation base), zero-initialised.
 * Protocol (all device side, CUDA-graph safe; `local_state` = 16 zero-initialised device-local bytes holding
 * the step counter and a CTA counter):
 *   - launch number s (1,2,...) of this entry writes slot s & 1: rank r's rows land at rows [r*rows, (r+1)*rows)
 *     of that slot on every rank;
 *   - before touching the slot, the kernel waits until flags[q] >= s-1 for every rank q IN ITS OWN MEMORY: rank q
 *     publishes s-1 only at the end of its launch s-1, which it enqueued after consuming the data of step s-2
 *     (CONTRACT: a rank consumes step k's gathered data on the launching stream before its launch k+1) -- so the
 *     slot is free.  With two slots this dependency is a whole step old: ranks never wait for each other inside a
 *     step (no barrier), they can drift by up to one step;
 *   - the last CTA to finish publishes s into flags[rank] of every rank with a system-scope release store after
 *     a system-scope fence; acr_b200_gather_wait (stream-ordered, tiny) returns once flags[q] >= s for all q in
 *     this rank's memory, i.e. the data of step s from every rank has landed here.  Rows >= the shard's count
 *     keep older data: validity is counts[q][2].
 * `rows` (per rank and slot) must be even and >= n_max; every rank must launch every step.                      */
typedef struct acr_b200_gather {
  uint64_t peer_base[8];      /* base address of every rank's allocation, as mapped into THIS process     */
  uint64_t multicast_base;    /* NVLS multicast mapping of the allocation, or 0                            */
  int32_t world, rank;
  int64_t rows;
  uint64_t slot_bytes;        /* multiple of 16                                                            */
  uint64_t counts_offset;     /* inside a slot, multiple of 16, >= world*rows*778*3*4                      */
  uint64_t flags_offset;      /* from the allocation base, multiple of 16, >= 2*slot_bytes                 */
  void* local_state;          /* device-local, 16 bytes, zero-initialised once                             */
} acr_b200_gather;

int acr_b200_mano_forward_gather(const float* model_l, const float* model_r, const float* poses,
                                 const float* betas, const int32_t* hand_type, int default_side,
                                 const int32_t* n_dev, int n_max, int center_idx, const float* cam,
                                 const float* offsets, float* verts, float* joints, float* center,
                                 float* verts_camed, float* pj2d, float* pj2d_org,
                                 const int32_t* counts_src, const acr_b200_gather* gather, void* stream);
/* Stream-ordered wait until the most recent gather launch of EVERY rank has landed in this rank's buffer. */
int acr_b200_gather_wait(const acr_b200_gather* gather, void* stream);

/* Backward of acr_b200_mano_forward for one side (the gradient of ManoLayer.forward, mano/manolayer.py:104-276,
 * which the reference gets from torch autograd): cotangents of verts / joints / center -> dposes, dbetas.
 *   model : packed model of `side` (0 left, 1 right); poses (n,48) WITHOUT the mean pose and betas (n,10): the
 *           values the forward saw.  Nothing is saved from the forward; the transforms are recomputed.
 *   center_idx : as in the forward (-1 none; a fingertip is ACR_B200_ENOTSUP).  With a centre, every vertex and
 *           joint had it subtracted and the centre is itself an output: d centre = dcenter - sum dverts - sum djoints.
 *   dverts (n,778,3), djoints (n,21,3), dcenter (n,3): cotangents, each may be NULL (= zero).
 *   workspace : acr_b200_mano_backward_workspace_floats(n) floats of caller-owned device scratch (per hand and
 *           vertex chunk: partial sums of the skinning-transform and blend-row cotangents); may be NULL when
 *           dverts and djoints are both NULL.
 * Outputs dposes (n,48) and dbetas (n,10); either may be NULL (not computed).  fp32; two launches; no atomics,
 * so repeated calls give bit-identical gradients.                                                      */
size_t acr_b200_mano_backward_workspace_floats(int n);
int acr_b200_mano_backward(const float* model, int side, const float* poses, const float* betas, int n,
                           int center_idx, const float* dverts, const float* djoints, const float* dcenter,
                           float* workspace, float* dposes, float* dbetas, void* stream);

/* ManoLayer.forward of one side with every pose input and root_palm (mano/manolayer.py:104-276), and its backward.
 *   pose_mode ACR_B200_POSE_AXISANG : pose (n,48) axis angles WITHOUT the mean pose, as acr_b200_mano_forward.
 *   pose_mode ACR_B200_POSE_ROTMAT  : pose (n,16,3,3) row-major matrices, unprojected (use_pca=False,
 *             joint_rot_mode='rotmat', :151-162).  Each is projected like batch_rotprojs (:436-453): Q = U V^T of
 *             its SVD M = U S V^T, column 2 negated when det Q < 0.  No mean pose is applied, as in the reference.
 *             Any matrix of rank >= 2 gives a finite orthogonal result; rank <= 1 is outside the contract (the
 *             reference's own result is arbitrary there) and gives NaN.  The gradient dpose (n,16,3,3) is the
 *             polar factor's: finite at exact rotations (where the SVD's derivative is not) and whenever no two
 *             singular values sum to zero.
 *   root_palm : nonzero => output joint 0 is the palm, (v95 + v22) / 2, instead of the wrist (:248-250).
 *   center_idx : as in acr_b200_mano_forward.  A fingertip, or the palm (0 with root_palm), is ACR_B200_ENOTSUP.
 *   betas (n,10).  Outputs verts (n,778,3) (16-byte aligned), joints (n,21,3), center (n,3); any may be NULL.
 * The backward takes the forward's arguments and the cotangents, and writes dpose (shaped like pose) and dbetas;
 * cotangents, workspace and outputs as in acr_b200_mano_backward.  A bad side, pose_mode or centre is
 * ACR_B200_EINVAL.  Axis angles without the palm make exactly the launches of acr_b200_mano_forward /
 * acr_b200_mano_backward.                                                                                     */
#define ACR_B200_POSE_AXISANG 0
#define ACR_B200_POSE_ROTMAT 1
int acr_b200_mano_layer_forward(const float* model, int side, const float* pose, int pose_mode, const float* betas,
                                int n, int center_idx, int root_palm, float* verts, float* joints, float* center,
                                void* stream);
int acr_b200_mano_layer_backward(const float* model, int side, const float* pose, int pose_mode,
                                 const float* betas, int n, int center_idx, int root_palm, const float* dverts,
                                 const float* djoints, const float* dcenter, float* workspace, float* dpose,
                                 float* dbetas, void* stream);

/* Forward-mode derivative (Jacobian-vector products) of acr_b200_mano_layer_forward, n_tan tangents per hand.
 *   model ... root_palm : as in acr_b200_mano_layer_forward (the same ACR_B200_ENOTSUP / EINVAL cases).
 *   tpose  : (n_tan, n, 48) or (n_tan, n, 16, 3, 3), tangents of pose; tbetas (n_tan, n, 10).  NULL = zero.
 *   verts, joints, center : the primal outputs, as in the forward; any may be NULL.
 *   tverts (n_tan, n, 778, 3), tjoints (n_tan, n, 21, 3), tcenter (n_tan, n, 3) : the output tangents, tangent-major;
 *            any may be NULL.  tcenter is zero without a centre.
 * In rotation-matrix mode the projection's tangent is the polar factor's, finite at exact rotations; at a zero axis
 * angle the Rodrigues tangent is finite too.  With verts and tverts both NULL only the 16 joints, the tips and the
 * palm are computed (one CTA per 8 hands and 4 tangents): a keypoint Jacobian costs no vertex pass.  fp32, no
 * atomics; a tangent's result does not depend on n_tan or on the other tangents, and repeated calls are
 * bit-identical.  n_tan < 0 is ACR_B200_EINVAL.                                                                */
int acr_b200_mano_layer_jvp(const float* model, int side, const float* pose, int pose_mode, const float* betas, int n,
                            int center_idx, int root_palm, int n_tan, const float* tpose, const float* tbetas,
                            float* verts, float* joints, float* center, float* tverts, float* tjoints, float* tcenter,
                            void* stream);

/* Camera translation of every hand from its 21 joints: the closed-form weighted least squares of
 * estimate_translation_np (acr/utils.py:430-472) -- the reference's own fall-back for the host-side
 * cv2.solvePnPRansac loop (estimate_translation :474-519, called from vertices_kp3d_projection :403-407,
 * SURVEY.md 8f-1).  joints_2d = (pj2d+1)*img_size/2 as in :404; a joint is used iff its pixel y > -2
 * and its z != -2 (:489-492); fewer than 4 usable joints -> (-1,-1,-1).  fp64 normal equations.
 * j3d (n,21,3), pj2d (n,21,2) -> cam_trans (n,3).  n_dev as in acr_b200_mano_forward.              */
int acr_b200_cam_trans(const float* j3d, const float* pj2d, const int32_t* n_dev, int n_max, float focal_length,
                       float img_size, float* cam_trans, void* stream);

/* Camera translation of every hand as the reference computes it: cv2.solvePnPRansac(SOLVEPNP_EPNP,
 * reprojectionError=20, iterationsCount=100) with K = [f 0 img_size/2; 0 f img_size/2; 0 0 1] on the usable
 * joints (the tests of acr_b200_cam_trans), in fp64 on the device, one warp per hand.  OpenCV's deterministic
 * RANSAC (its RNG, 5-point EPnP hypotheses, fp32 reprojection test) and the final EPnP on all inliers.
 *   fewer than 4 usable joints  -> (-1,-1,-1), as acr_b200_cam_trans;
 *   exactly 4                   -> acr_b200_cam_trans's least squares (OpenCV would run P3P: a deviation);
 *   exactly 5                   -> one EPnP, every joint an inlier (OpenCV skips RANSAC there);
 *   no RANSAC consensus         -> acr_b200_cam_trans's least squares (the reference's except-branch).
 * inlier_mask (n) int32, optional (NULL skips it): bit j set iff joint j is an inlier of the final fit; 0 where
 * the result is the least squares or (-1,-1,-1).  n_dev as in acr_b200_mano_forward; rows >= *n_dev are not
 * written.  No allocation, no host synchronisation, no atomics: graph-capturable.                       */
int acr_b200_cam_trans_pnp(const float* j3d, const float* pj2d, const int32_t* n_dev, int n_max, float focal_length,
                           float img_size, float* cam_trans, int32_t* inlier_mask, void* stream);

/* Frame pre-processing on the device (SURVEY.md 8f-2): n BGR frames (n,H,W,3) -> RGB, white (255) pad to a
 * `side` x `side` square (pad_t rows above, pad_l columns left), bicubic resize to out_size x out_size.
 * Replaces img_preprocess / process_image_ori / image_pad_white_bg + cv2.resize(INTER_CUBIC)
 * (acr/utils.py:1303-1337).  Integer arithmetic of OpenCV's generic 8-bit cubic path (11-bit coefficients,
 * replicate border, (sum + 2^21) >> 22); the (out_size,4) int16 coefficient and (out_size) int32 offset
 * tables come from acr_b200/preprocess.py::cubic_tables (host, float32 like OpenCV).                   */
int acr_b200_preprocess(const uint8_t* frames_bgr, int n, int H, int W, const int16_t* coef_x,
                        const int32_t* ofs_x, const int16_t* coef_y, const int32_t* ofs_y, int side, int pad_t,
                        int pad_l, int out_size, uint8_t* out_rgb, void* stream);

/* The cubic tables of acr_b200/preprocess.py::cubic_tables on the device, for n source squares at once: frame i
 * (side n_src[i], device int32) gets coef[i] (out_size,4) int16 and ofs[i] (out_size) int32, bit for bit the host's
 * float32 arithmetic (explicit round-to-nearest operations, no contraction).  One thread per (frame, d).  An
 * n_src[i] < 1 gives zero tables.  Graph-capturable: a replay reads the sides it finds in n_src.            */
int acr_b200_cubic_tables(const int32_t* n_src, int n, int out_size, int16_t* coef, int32_t* ofs, void* stream);

/* One frame of a ragged batch: its BGR HWC bytes start `offset` bytes into the packed buffer; it is white-padded
 * to a side x side square with pad_t rows above and pad_l columns to the left. 32 bytes. */
typedef struct acr_b200_frame {
  int64_t offset;
  int32_t H, W, side, pad_t, pad_l;
  int32_t reserved;  /* 0 */
} acr_b200_frame;

/* acr_b200_preprocess for n frames of any sizes in one launch (grid: pixel blocks x n).  `frames_bgr` holds
 * src_bytes bytes: every frame back to back (HWC, contiguous), where frames[i] (device) says.  coef (n,out_size,4)
 * and ofs (n,out_size) are frame i's tables for its side (acr_b200_cubic_tables), used on both axes.  Per-pixel
 * arithmetic as acr_b200_preprocess.  Outputs out_rgb (n,out_size,out_size,3) and, when offsets is not NULL, the
 * (n,10) fp32 offsets vectors [side, side, 0,0,0,0, pad_t, r, b, pad_l] of the descriptors.
 * n < 1 or > 65535, out_size < 1, src_bytes < 0 or a NULL input is ACR_B200_EINVAL.  The descriptors are device
 * data (a graph replay may change every frame's size), so they are checked on the device: a frame that breaks
 * H, W >= 1, side = max(H, W), pad_t, pad_l >= 0, pad_t + H <= side, pad_l + W <= side, offset >= 0 or
 * offset + H*W*3 <= src_bytes reads nothing and gets an all-zero image and offsets row.                  */
int acr_b200_preprocess_ragged(const uint8_t* frames_bgr, int64_t src_bytes, const acr_b200_frame* frames, int n,
                               const int16_t* coef, const int32_t* ofs, int out_size, uint8_t* out_rgb,
                               float* offsets, void* stream);

/* Part labels: SegmNet's 33-class logits -> one uint8 label per pixel of each frame (0 background, 1-16 right-hand
 * parts, 17-32 left-hand parts; the network's channel order).  segms: n maps of map_size x map_size pixels, NHWC with
 * pix_stride elements per pixel (the arena's `segms`: 48), dtype ACR_DT_BF16 / ACR_DT_F16 / ACR_DT_F32, channels
 * 0..32 the logits, 16-byte aligned.  offsets (n,10) fp32 on the device: image i's row [side, side, 0,0,0,0, pad_t,
 * pad_r, pad_b, pad_l] (the pj2d_org offsets) gives its frame of H = side - pad_t - pad_b rows and W = side - pad_l -
 * pad_r columns, and
 *   labels_i[y, x] = argmax_c bilinear(segms_i[c], side)[y + pad_t, x + pad_l]
 * with F.interpolate(size=(side, side), mode='bilinear', align_corners=False) weights, interpolated in fp32, ties to
 * the lowest channel (tests/part_labels_ref.py is the statement).  Frame i's H*W bytes start frame_offset[i] bytes
 * into `labels`: the exclusive prefix of H*W over the frames before it (a flagged frame counts 0 when its geometry is
 * invalid).  flags[i] (int32): ACR_B200_PART_LABELS_INVALID when the row has a negative or non-integer entry, unequal
 * sides, a side outside 1..ACR_B200_PART_LABELS_MAX_SIDE, pad_t + pad_b >= side or pad_l + pad_r >= side;
 * ACR_B200_PART_LABELS_OVER_CAPACITY when its labels would end past `capacity` bytes; 0 otherwise.  A flagged frame
 * gets no stores.  The geometry is read on the device and the grids depend on n and map_size only, so a graph replay
 * may change every frame's size.  Two launches (the prefix, then one CTA per 16 x 16 source quads and image); no
 * atomics, the same bytes on every call.  A NULL argument, another dtype, a stride that does not cover 33 channels in
 * 16-byte loads, n outside 1..65535, map_size outside 1..4096 or capacity < 0 is ACR_B200_EINVAL.                  */
#define ACR_B200_PART_LABELS_MAX_SIDE 16384
#define ACR_B200_PART_LABELS_INVALID 1
#define ACR_B200_PART_LABELS_OVER_CAPACITY 2
int acr_b200_part_labels(const void* segms, int dtype, int pix_stride, int map_size, const float* offsets, int n,
                         int64_t capacity, uint8_t* labels, int64_t* frame_offset, int32_t* flags, void* stream);

/* Multi-hand tracking of one stream between parse and MANO: a stable track id per detected hand and one OneEuro
 * bank per track, for up to K hands per side (the parse's max_hands_per_side).  The filter replaces OneEuroFilter /
 * LowPassFilter (acr/utils.py:1485-1527), smooth_results (:1478-1482), smooth_global_rot_matrix (:1466-1470) and the
 * per-frame host loop of acr/main.py:69-83 (SURVEY.md 8f-3): K = 1 with the gate open (>= 90) and no miss limit
 * (max_missed = 2^31 - 1) is the reference's per-hand-type smoothing, one bank per side.  The B images of a call are B
 * consecutive frames in time order; rows are in the parse's layout (row_src (n,4): image, side, flat centre cell
 * y*64+x, unused).  Per frame and side: live tracks match detections greedily by integer squared cell distance
 * within `gate` cells (ties by slot, then row); a track unmatched for more than `max_missed` consecutive frames
 * ends; an unmatched detection starts a track in the lowest free slot, or replaces the most-missed unmatched one.
 * Track ids are 2*c + side with a per-side birth counter c, never reused.  tests/track_ref.py is the statement.
 * track_id (n_max) gets each row's id, -1 for a row that is no detection (detection_flag <= 0, at or past *n_dev,
 * out of range, or out of time order -- such rows are left untouched).  With poses (n,48) and betas (n,10), each
 * tracked detection is filtered in place through its track's bank with that filter (a track's first frame passes
 * the pose's 45 values and the betas through); with both NULL only ids are computed.
 * `state`: device buffer of acr_b200_track_state_bytes(K) bytes, zeroed = no tracks.  One launch over B frames
 * equals B launches of one frame, bit for bit.  K outside 1..16, B < 1, n_max outside 0..2*K*B, gate or max_missed
 * < 0, a NULL state / row_src / track_id, exactly one of poses and betas NULL, or smooth_coeff <= 0 with poses is
 * ACR_B200_EINVAL and nothing is launched.  acr_b200_track_state_bytes returns 0 for K outside 1..16.          */
size_t acr_b200_track_state_bytes(int K);
int acr_b200_track_hands(float* poses, float* betas, const int32_t* row_src, const float* detection_flag,
                         const int32_t* n_dev, int n_max, int B, int K, int gate, int max_missed, float smooth_coeff,
                         void* state, int32_t* track_id, void* stream);

/* Multi-hand tracking of up to S streams in one batch: acr_b200_track_hands per stream, with the streams' frames
 * interleaved in any way.  frame_stream (B) int32 on the device gives the stream slot of each image, in 0..S-1; the
 * images of one stream are its frames in time order, in ascending batch index.  For every stream s the result is
 * acr_b200_track_hands run on s's frames alone, bit for bit: the rows of s's images in their table order, the images
 * renumbered 0..B_s-1 in batch order, and slot s of the state.  So each rule of the single-stream call (detections,
 * malformed, out-of-range and out-of-time-order rows, ids 2*c + side with a birth counter per stream and side)
 * applies per stream, and the key of a track is (stream, id).  A frame whose stream is outside 0..S-1 is not tracked:
 * its rows get id -1 and stay untouched.  frame_begin (B) int32 on the device, or NULL: a nonzero entry zeroes the
 * frame's stream slot just before that frame, as a zeroed single-stream state (a new camera in that slot); which
 * rows are detections is still decided over the stream's rows of the whole call, as one single-stream call does.
 * `state`: S consecutive slots of acr_b200_track_state_bytes(K) bytes; slot s is byte for byte a single-stream state,
 * so one can be copied in or out as it is.  `workspace`: acr_b200_track_streams_workspace_bytes(n_max, B, S) bytes of
 * caller-owned device scratch (the per-stream bucketing of frames and rows).  The launches depend on B, K and S only:
 * no host sync, capturable in a CUDA graph.  The checks of acr_b200_track_hands, S outside 1..4096, or a NULL
 * frame_stream or workspace is ACR_B200_EINVAL and nothing is launched.  The workspace size is 0 for n_max < 0, B < 1
 * or S outside 1..4096.  tests/stream_track_ref.py is the statement.                                           */
size_t acr_b200_track_streams_workspace_bytes(int n_max, int B, int S);
int acr_b200_track_streams(float* poses, float* betas, const int32_t* row_src, const float* detection_flag,
                           const int32_t* n_dev, int n_max, int B, int K, int gate, int max_missed, float smooth_coeff,
                           void* state, int32_t* track_id, const int32_t* frame_stream, const int32_t* frame_begin,
                           int S, void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------
 * Rotations
 * ---------------------------------------------------------------------------------------- */
/* rot6D_to_angular (acr/utils.py:378-382): n_rot 6-vectors -> n_rot axis-angle 3-vectors,
 * through Gram-Schmidt (:362-376), 4-case quaternion (:826-906), atan2 (:773-823), NaN->0. */
int acr_b200_rot6d_to_aa(const float* rot6d, int n_rot, float* aa, void* stream);
/* batch_rodrigues (mano/manolayer.py:423-434): n axis-angle -> n row-major 3x3.            */
int acr_b200_rodrigues(const float* aa, int n_rot, float* rotmat, void* stream);

/* ------------------------------------------------------------------------------------------
 * Centre parsing + parameter sampling
 * ---------------------------------------------------------------------------------------- */
typedef struct acr_b200_map {      /* one fp32 NHWC map: element (b,y,x,c) at              */
  const float* ptr;                /* ptr[((b*H + y)*W + x)*pix_stride + c]                */
  int pix_stride;
} acr_b200_map;

typedef struct acr_b200_parse_out {
  /* compacted rows, left hands first (all images in order) then right hands; capacity 2*B */
  float* params_pred;        /* (2B,109) */
  float* cam;                /* (2B,3)   */
  float* global_orient;      /* (2B,3)   axis-angle */
  float* hand_pose;          /* (2B,45)  axis-angle */
  float* betas;              /* (2B,10)  */
  float* poses;              /* (2B,48)  = [global_orient | hand_pose] */
  float* detection_flag;     /* (2B)     1.0 / 0.0 */
  int64_t* reorganize_idx;   /* (2B)     meta batch id of the row's image */
  int64_t* batch_ids;        /* (2B)     local image index of the row */
  int64_t* centers_pred;     /* (2B,2)   [x,y] on the 64-grid, rows as above */
  float* centers_conf;       /* (2B)     raw centre-map value at the centre */
  int32_t* hand_type;        /* (2B)     0 left, 1 right */
  float* offsets_out;        /* (2B,10)  offsets row of the image, or NULL */
  int32_t* counts;           /* (8) [0]=L, [1]=R, [2]=L+R, [3]=#true detections, [4]=#left, [5]=#right */
  /* dense per-image scratch, (B,2): flat index and score of the top-1 centre of each side */
  int32_t* top_idx;
  float* top_score;
  int32_t* row_src;          /* (2B,4) scratch: image, side, flat index, other side's index | -1 */
} acr_b200_parse_out;

/* ResultParser.parse (acr/result_parser.py:21-40) = parse_maps (:85-190) with K=1 centre
 * extraction (:218-249), parameter sampling (:49-57), cross-hand prior (:141-145) gated by
 * determine_coeff (:42-47), then rot6D_to_angular on global_orient / hand_pose.
 * B images, H=W=64 maps.  meta_batch_ids (B) int64 may be NULL (=> arange), offsets (B,10)
 * may be NULL.  All batch>1 quirks of the reference are reproduced (see oracle/parse_ref.py). */
int acr_b200_parse(acr_b200_map l_center, acr_b200_map r_center, acr_b200_map l_params,
                   acr_b200_map r_params, acr_b200_map l_prior, acr_b200_map r_prior, int B,
                   float conf_thresh, const int64_t* meta_batch_ids, const float* offsets,
                   acr_b200_parse_out out, void* stream);

/* Multi-hand parsing: up to K hands per image and side, the reference's train_flag=True centre selection
 * (acr/result_parser.py:218-243 with max_hand = K).  Per image and side: the 5x5 max-pool NMS of acr_b200_parse,
 * the top K scores in descending order (equal scores: lower flat index first), kept while score > conf_thresh.
 * Rows: every left hand (image-major, rank-minor), then every right hand; a side with no detection in the batch
 * gets the dummy row of acr_b200_parse.  The cross-hand prior of hand (b, side, k) is its own side's prior map
 * sampled at the nearest opposite-side hand of image b (integer squared grid distance, ties to the lower rank),
 * nothing when image b has none; the batch-global determine_coeff gate uses the first left and first right rows.
 * K = 1 gives acr_b200_parse's outputs bit for bit.  Capacities: every row buffer of `out` holds 2*K*B rows,
 * top_idx / top_score are (B,2,K), row_src is (2*K*B,4); counts has the meaning above.
 * K outside 1..16 is ACR_B200_EINVAL. */
int acr_b200_parse_topk(acr_b200_map l_center, acr_b200_map r_center, acr_b200_map l_params,
                        acr_b200_map r_params, acr_b200_map l_prior, acr_b200_map r_prior, int B, int K,
                        float conf_thresh, const int64_t* meta_batch_ids, const float* offsets,
                        acr_b200_parse_out out, void* stream);

/* ------------------------------------------------------------------------------------------
 * Network launch plan (backbone + heads)
 * ---------------------------------------------------------------------------------------- */
enum {
  ACR_OP_STEM = 1,        /* uint8 NHWC image -> x/255*2-1 -> conv3x3 s2 + BN + ReLU           */
  ACR_OP_CONV = 2,        /* implicit-GEMM NHWC conv (k in {1,3}, s in {1,2}) on wgmma          */
  ACR_OP_FUSE = 3,        /* relu(sum_i nearest_up(term_i, 2^shift_i)), fp32 accumulation       */
  ACR_OP_BILINEAR2X = 4,  /* F.interpolate(x2, bilinear, align_corners=True)                    */
  ACR_OP_COORD = 5,       /* write the two coord-conv channels                                  */
  ACR_OP_POOL = 6,        /* Hadamard_product: softmax over HW x feature matmul (partials)      */
  ACR_OP_PARTHEAD = 7,    /* merge partials + LocallyConnected2d + Linear + per-image bias      */
  ACR_OP_CONV_REF = 8,    /* debug: same contract as ACR_OP_CONV on CUDA cores (tests only)     */
  ACR_OP_FINALCONV = 9,   /* (retired)                                                          */
  ACR_OP_IM2COL_STEM = 10, /* uint8 NHWC image -> 3x3 s2 im2col of x/255*2-1, 27(+5 zero) 16-bit channels */
  ACR_OP_STEM_TC = 11,     /* STEM on the tensor cores: the im2col operand is built in shared memory, never in HBM   */
  ACR_OP_MAXPOOL = 12      /* nn.MaxPool2d(3, stride 2, padding 1) on 16-bit NHWC (ResNet trunk)                     */
};  /* kinds stay below 16: acr_b200_plan_profile indexes ms_by_kind[16] */
enum { ACR_CONV_BIAS_PER_IMAGE = 1, ACR_CONV_POW11_CH0 = 2, ACR_CONV_XPAIR = 4, ACR_CONV_S2X = 8, ACR_CONV_EXTRA = 16,
       ACR_CONV_DECONV = 32, ACR_CONV_BLOCK = 64, ACR_CONV_BLOCK_MID = 128, ACR_CONV_BOTTLENECK = 256 };
enum { ACR_DT_BF16 = 0, ACR_DT_F16 = 1, ACR_DT_F32 = 2, ACR_DT_U8 = 3,
       ACR_DT_TF32 = 4 /* an act_dtype only (plan_create, run_op, pack_conv): fp32 storage, tf32 tensor-core convs */ };

typedef struct acr_b200_tensor {  /* NHWC activation inside the arena (per-image extents)  */
  uint64_t offset;                /* byte offset of element (0,0,0,0) from the arena base   */
  int32_t C, H, W;                /* logical channels (multiple of 8 for 16-bit types)      */
  int32_t pix_stride;             /* elements between neighbouring pixels (>= C)            */
  int32_t dtype;
  int32_t external;               /* 1: `offset` is relative to the external-input pointer  */
} acr_b200_tensor;

/* One launch.  Which fields are read depends on `kind`:
 *  STEM      in[0]=image(u8,external) out; w_offset[0]=fp32 [27][64] folded weights, [1]=fp32 bias[64]
 *  STEM_TC   in[0]=image(u8,external) out (64 ch, H/2 x W/2, 16-bit); w_offset[0]=packed [64][32] 16-bit weights (input
 *            channel (ky*3+kx)*3+ci, 27..31 zero, BN folded), [1]=fp32 bias[64]: conv1 + bn1 + ReLU of acr/model.py:832-835
 *            as one wgmma GEMM whose A operand (the 27 normalised taps of every output pixel) is built in shared memory.
 *            k = 7: the ResNet stem instead, conv1 7x7 stride 2 padding 3 (3 -> 64) + bn1 + ReLU; w_offset[0] = packed
 *            [64][160] (input channel (ky*7+kx)*3+ci, 147..159 zero, BN folded).  Any other k (0 included) = 3x3.
 *            Both forms pad with zeros (not -1) and carry the bias in spare K channels.  The output tiles per row and
 *            per image must be powers of two.
 *  MAXPOOL   in[0] (16-bit NHWC, C and pix_stride multiples of 8) -> out (H/2 x W/2, same dtype): max over the
 *            valid taps of the 3x3 window at (2y-1.., 2x-1..) (padding never wins, as nn.MaxPool2d(3, 2, 1))
 *  IM2COL_STEM in[0]=image(u8,external) out (32 ch, H/2 x W/2): channel (ky*3+kx)*3+ci = normalised tap,
 *            0 outside the image; the stem conv then runs as a 1x1 CONV on the tensor cores
 *  CONV(_REF) in[0]=x, in[1]=residual (has_residual) out; w_offset[0]=packed 16-bit weights
 *            [cout_pad][k*k][cin_pad], w_offset[1]=fp32 bias[cout_pad]; shift[0] = flag bits:
 *            ACR_CONV_BIAS_PER_IMAGE (bias = fp32 (B,cout_pad) tensor aux[0] in the arena instead of
 *            w_offset[1]) | ACR_CONV_POW11_CH0 (output channel 0 -> 1.1**x, acr/model.py:95-96)
 *            | ACR_CONV_XPAIR (3x3 s1 64->64 whose weights are the x-paired expansion of a 32->32 conv: channel =
 *            (x parity)*32 + c on a W/2 grid; the kx=0 / kx=2 taps are non-zero only in the [N 0..31][K 32..63] /
 *            [N 32..63][K 0..31] corner, which is all the kernel multiplies)
 *            | ACR_CONV_EXTRA (in[1..n_in) are further terms of the same shape class as `out`, term j nearest-upsampled by
 *            2**shift[j]: out = act(conv(in[0]) + bias + sum of terms) -- the fuse sum of HighResolutionModule.forward
 *            (acr/model.py:677-684) folded into the conv that produces one of its terms; no residual then)
 *            | ACR_CONV_S2X (3x3 STRIDE-2 conv of a dense 32-channel tensor: in[0] is its x-paired view (H, W/2, 64) --
 *            even pixel's channels then the odd neighbour's in one 128-byte row -- `out` is (H/2, W/2); the packed
 *            weights [cout_pad][9][64] carry the 32 input channels of tap (ky,kx) at K offset 32*(kx != 1))
 *            | ACR_CONV_DECONV (nn.ConvTranspose2d(kernel 4, stride 2, padding 1, no bias) + BN (+ReLU): k = 4,
 *            stride = 2, `out` is (2H, 2W), cin_pad a multiple of 64, no residual / extra terms.  Output pixel
 *            (2m+py, 2n+px) is a 2x2 conv of the input at row offsets {-1, 0} (py = 0: ky = 3, 1) or {0, +1} (py = 1:
 *            ky = 2, 0), the same along x.  The packed weights are [4 parities py*2+px][cout_pad][4 taps ty*2+tx]
 *            [cin_pad], tap (ty,tx) of parity (py,px) = w[ci][co][3-py-2ty][3-px-2tx] of the (cin, cout, 4, 4)
 *            ConvTranspose2d weight, BN folded; w_offset[1] = fp32 bias[cout_pad].  Output rows may be a channel slice
 *            of a wider buffer (pix_stride >= cout_pad).)
 *            | ACR_CONV_BLOCK (this conv and the NEXT op are one HRNet BasicBlock: both 3x3 stride-1 64->64 with ReLU, or
            both x-paired; the next op reads this op's output, has this op's input as its residual and is the only reader
            of this op's output.  The plan runs the pair as ONE launch whose intermediate stays in shared memory
            (csrc/conv_block.cuh); bit-identical to two launches.  ACR_B200_FUSE_BLOCKS=0 in the environment at plan
            creation ignores the flag)  | ACR_CONV_BLOCK_MID (with ACR_CONV_BLOCK: the fused launch still writes this
            op's output, for readers outside the plan)
            | ACR_CONV_BOTTLENECK (this conv and the NEXT TWO ops are one Bottleneck: this op a 1x1 stride-1 C_in -> 64 conv
            with ReLU, C_in = 64 or 256; the next a 3x3 stride-1 64 -> 64 conv with ReLU on this op's output; the one after
            a 1x1 stride-1 64 -> 256 conv with ReLU on that output, whose residual is any 256-channel tensor of the same
            grid (the block input, or the downsample's output).  Both intermediates have no reader outside the triple and
            are not written.  The three ops sit on one stream, and the second and third wait for nothing this op does
            not.  The plan runs the triple as ONE launch (csrc/conv_bottleneck.cuh); bit-identical to three launches.
            ACR_B200_FUSE_BLOCKS=0 at plan creation ignores this flag too)
            Contracts of the tensor-core CONV: k in {1, 3} (4 with ACR_CONV_DECONV), stride in {1, 2}; a 1x1
 *            stride-2 conv (ResNet downsample, padding 0) reads input pixel (2y, 2x); cin_pad and cout_pad are
 *            multiples of 16 up to 2048 (K per tap up to 2048, N up to 2048 as 16 balanced virtual tiles of 128).
 *            The fp32 validation plan and CONV_REF take neither ACR_CONV_DECONV, MAXPOOL nor the k = 7 stem:
 *            they return ACR_B200_ENOTSUP.
 *  FUSE     in[0..n_in) with shift[i]; out
 *  BILINEAR2X / COORD (fparam unused; COORD writes channels [in[0].C, pix_stride) of `out`)
 *  POOL      in[0]=contact features (256ch), in[1]=segm logits; out = partials (fp32, 1x1xC)
 *  PARTHEAD  in[0]=partials; out=pooled (fp32 256*32); aux[0..1]=bias_img l,r (112); aux[2..3]=
 *            pare l,r (106); w_offset[0..1]=LC weights l,r; [2],[3]=shape conv w,b; [4..5]=Linear w
 *            l,r; [6..7]=Linear b; [8..9]=final conv w (109,218) l,r; [10..11]=final conv b
 *  FINALCONV (retired: the folded contact_layers[4|5] conv now runs as a CONV with
 *            ACR_CONV_BIAS_PER_IMAGE on the tensor cores)                                  */
typedef struct acr_b200_op {
  int32_t kind;
  int32_t n_in;
  acr_b200_tensor out;
  acr_b200_tensor in[4];
  acr_b200_tensor aux[4];
  uint64_t w_offset[12];          /* byte offsets into the weight blob                      */
  int32_t k, stride, relu, has_residual;
  int32_t cin_pad, cout_pad;      /* K per tap / N, multiples of 16                         */
  int32_t shift[4];
  int32_t stream_id;              /* plan-internal stream (branch-level concurrency)        */
  int32_t wait_mask;              /* bit i: wait for the last op recorded on stream i       */
  float fparam[4];
} acr_b200_op;

typedef struct acr_b200_plan acr_b200_plan;

/* Build a launch plan for `batch` images.  `arena` (device, `arena_bytes`) holds every
 * activation; `weights` (device) the packed weight blob; ops are copied.  Creates the TMA
 * tensor maps and internal streams/events.  Replaces the module tree construction +
 * forward dispatch of acr/model.py:23-65 (ACR), :691-865 (HigherResolutionNet).
 * act_dtype:
 *   ACR_DT_BF16 / ACR_DT_F16  the product plans: 16-bit activations and weights, fp32 accumulation on the tensor cores.
 *   ACR_DT_F32                the validation plan: fp32 storage, fp64 accumulation on the CUDA cores (every op).
 *   ACR_DT_TF32               the TF32 plan -- what an fp32 PyTorch model runs on Ampere / Hopper with cuDNN's default
 *                             allow_tf32: fp32 storage (tensor records still say ACR_DT_F32) and fp32 outputs, every
 *                             ACR_OP_CONV on the wgmma tensor cores with tf32 operands and fp32 accumulation.  Weights
 *                             come from acr_b200_pack_conv(..., ACR_DT_TF32); the kernel rounds activations to the nearest
 *                             tf32 in shared memory (storage stays fp32).  Every other
 *                             op (stem, fuse, bilinear, coord, pooling, CONV_REF) runs on the validation plan's kernels,
 *                             the part head as in every plan.  ACR_CONV_BLOCK and ACR_CONV_BOTTLENECK marks are ignored (the
 *                             resident fp32 weight sets do not fit the fused kernels' shared memory), and the x-paired, stride-2 x-paired
 *                             and transposed conv forms are ACR_B200_EINVAL.
 * A tensor record whose dtype is ACR_DT_TF32 is ACR_B200_EINVAL (here and in acr_b200_run_op).                           */
int acr_b200_plan_create(const acr_b200_op* ops, int n_ops, int batch, void* arena,
                         size_t arena_bytes, const void* weights, size_t weight_bytes,
                         int act_dtype, acr_b200_plan** plan_out);
/* Run the plan on `stream`: `image` is the external uint8 (batch,512,512,3) input.        */
int acr_b200_plan_run(acr_b200_plan* plan, const void* image, void* stream);
/* Like plan_run, but brackets every launch with CUDA events on `stream` (serialising the plan) and
 * accumulates device milliseconds / launch counts per op kind into ms_by_kind[16] / n_by_kind[16]
 * (host arrays, indexed by ACR_OP_*).  Synchronises `stream`.  Used by bench.py for the roofline. */
int acr_b200_plan_profile(acr_b200_plan* plan, const void* image, void* stream, float* ms_by_kind,
                          int32_t* n_by_kind);
/* The same serialised, event-bracketed pass, but writes the device milliseconds of op i into ms_by_op[i]
 * (host array of n_ops floats, in plan order; a fused BasicBlock's or Bottleneck's time is on its first conv, the others
 * read 0).
 * Synchronises `stream`.  Per-layer tables.                                                 */
int acr_b200_plan_profile_ops(acr_b200_plan* plan, const void* image, void* stream, float* ms_by_op);
/* Number of kernel launches one plan_run issues (for bench.py's gpu_launches): the plan's ops less the
 * second convs of fused BasicBlocks (ACR_CONV_BLOCK) and the second and third of fused Bottlenecks (ACR_CONV_BOTTLENECK). */
int acr_b200_plan_num_launches(const acr_b200_plan* plan);
/* launch_of_op[i] (host array of n_ops int32) = index of the launch that computes op i: the two convs of a fused
 * BasicBlock, and the three of a fused Bottleneck, share one launch.                                                              */
int acr_b200_plan_op_launch(const acr_b200_plan* plan, int32_t* launch_of_op);
void acr_b200_plan_destroy(acr_b200_plan* plan);

/* Single-op entry used by the parity tests (same code path as inside a plan, any act_dtype of plan_create).      */
int acr_b200_run_op(const acr_b200_op* op, int batch, void* arena, const void* weights,
                    const void* external, int act_dtype, void* stream);

/* Host-side weight folding/packing for one conv (acr_b200_weights_pack of SURVEY.md 8b):
 * folds eval-mode BatchNorm (acr/model.py BN after every conv) into w/b and repacks
 * OIHW fp32 -> [cout_pad][kh][kw][cin_pad] 16-bit (K-major rows for the wgmma B operand),
 * or fp32 for ACR_DT_F32 and ACR_DT_TF32.  ACR_DT_TF32 packs exactly like ACR_DT_F32, then
 * rounds every weight to the nearest tf32 value (ties away from zero, as cvt.rna.tf32.f32):
 * its low 13 mantissa bits are zero.  The bias is fp32 in every mode.
 * bn_* may be NULL (no BN); conv_bias may be NULL.  All pointers are HOST pointers.       */
int acr_b200_pack_conv(const float* w_oihw, const float* conv_bias, const float* bn_gamma,
                       const float* bn_beta, const float* bn_mean, const float* bn_var, float bn_eps,
                       int cout, int cin, int k, int cout_pad, int cin_pad, int act_dtype,
                       void* w_packed_host, float* bias_host);

/* ---- JPEG decoding (csrc/jpeg.cu) ------------------------------------------------------------------
 * Replaces the host decode of every input mode of the reference (cv2.imread in image / folder mode, and the
 * read-back of the frames split_frame writes in video mode; /root/reference/demo.py, acr/utils.py).  The host parses
 * the headers (acr_b200/jpeg.py) into one acr_b200_jpeg_frame per file; the entropy-coded segments travel
 * untouched, packed back to back.  Output: BGR HWC frames packed back to back, equal to cv2.imdecode(buf,
 * IMREAD_COLOR) (libjpeg-turbo: JDCT_ISLOW, fancy upsampling) byte for byte.                                      */
#define ACR_B200_JPEG_CHUNK 256  /* entropy-coded bytes per decoder thread */
#define ACR_B200_JPEG_MAX_SCAN_BYTES (1 << 28)  /* coded_len must be below this: positions are int32 bit offsets */

/* A Huffman table in lookup form.  1424 bytes. */
typedef struct acr_b200_jpeg_huff {
  uint16_t lut[512];   /* next 9 bits -> (code length << 8) | symbol; 0 when the code is longer than 9 bits */
  int32_t maxcode[18]; /* largest code of each length 1..16, -1 if none; [17] = INT32_MAX */
  int32_t valoff[18];  /* symbol of code c of length l = huffval[c + valoff[l]] */
  uint8_t huffval[256];
} acr_b200_jpeg_huff;

/* One file of a batch.  Component c's plane is comp_bw[c] x comp_bh[c] blocks (whole MCUs); its blocks start at
 * block coef_offset + comp_block0[c] of the workspace.  Block k of an MCU belongs to component slot_comp[k], at
 * (slot_dy[k], slot_dx[k]) inside the MCU.  chunk_begin / block_begin: the frame's first chunk (of
 * ACR_B200_JPEG_CHUNK coded bytes) and block in the batch's numbering.  9112 bytes. */
typedef struct acr_b200_jpeg_frame {
  int64_t coded_offset; /* entropy-coded segment: bytes [coded_offset, coded_offset + coded_len) of `coded` */
  int64_t out_offset;   /* first BGR byte of the frame in `out_bgr` */
  int64_t coef_offset;  /* = block_begin */
  int32_t coded_len, H, W, ncomp;
  int32_t mcus_x, mcus_y, bpm, restart; /* blocks per MCU; restart interval in MCUs, 0 = none */
  int32_t chunk_begin, n_chunks, block_begin, n_blocks;
  int32_t comp_h[3], comp_v[3];   /* sampling factors (grey: 1, 1) */
  int32_t comp_bw[3], comp_bh[3]; /* plane size in blocks */
  int32_t comp_w[3], comp_hgt[3]; /* component size in samples (libjpeg's downsampled_width / _height) */
  int32_t comp_block0[3];
  int32_t n_scans; /* 0: a single-scan file; > 0: a multi-scan file decoded from that many acr_b200_jpeg_scan
                      descriptors (acr_b200_jpeg_decode_scans only): the MCU geometry above is the frame's, restart
                      and the Huffman tables are unused, and the chunk and coded ranges cover its scans' ranges */
  int8_t slot_comp[8], slot_dy[8], slot_dx[8];
  uint16_t quant[3][64]; /* natural order */
  acr_b200_jpeg_huff dc[3], ac[3];
} acr_b200_jpeg_frame;

/* Status bits of acr_b200_jpeg_decode, per frame (0 = decoded). */
#define ACR_B200_JPEG_BAD_CODE 1     /* a code that is not in the table, or an AC run past the block */
#define ACR_B200_JPEG_TRUNCATED 2    /* the segment ends before the last MCU */
#define ACR_B200_JPEG_BAD_RESTART 4  /* a restart marker out of place or out of sequence */
#define ACR_B200_JPEG_BAD_MARKER 8   /* another marker inside the entropy-coded data */
#define ACR_B200_JPEG_BAD_LENGTH 16  /* more coded blocks than the frame has */

/* Workspace of acr_b200_jpeg_decode for at most max_chunks chunks and max_blocks blocks over the batch. */
size_t acr_b200_jpeg_workspace_bytes(int64_t max_chunks, int64_t max_blocks);
/* Byte offset in that workspace of the coefficient blocks, which stay valid after a decode: block k of the batch
 * (frame.coef_offset + comp_block0[c] + row * comp_bw[c] + column) is 64 int16 quantised coefficients in natural
 * order, DC included.  Frames with status != 0 have undefined coefficients. */
size_t acr_b200_jpeg_coef_offset(int64_t max_chunks);

/* Decode n frames (frames: device descriptors) from `coded` (coded_bytes bytes) into `out_bgr` (out_bytes bytes),
 * in a fixed number of launches: speculative Huffman decoding (one thread per chunk, started at a guessed code
 * boundary), one CTA per frame to synchronise the chunks and prefix their block counts and DC predictions, the
 * coefficient stores, the islow IDCT, and fancy upsampling with colour conversion.  Grids are sized by max_chunks,
 * max_blocks and out_bytes; the device skips work past the batch's real totals, so a CUDA graph can replay it with
 * other files.  status (device, n int32) gets each frame's ACR_B200_JPEG_* bits; a frame with status != 0 gets an
 * all-black image (none when its descriptor does not fit the buffers, status bit 256).  Every read stays inside the
 * frame's segment, and every store inside its own output.
 * Frames whose descriptor has ncomp == 0 are skipped (left untouched in out_bgr, status 0); a multi-scan frame
 * (n_scans != 0) gets status 256 here (acr_b200_jpeg_decode_scans decodes it).                                   */
int acr_b200_jpeg_decode(const uint8_t* coded, int64_t coded_bytes, const acr_b200_jpeg_frame* frames, int n,
                         int64_t max_chunks, int64_t max_blocks, void* workspace, size_t workspace_bytes,
                         uint8_t* out_bgr, int64_t out_bytes, int32_t* status, void* stream);

/* One scan of a progressive (SOF2) or multi-scan sequential (SOF0 / SOF1) file.  Scans of one frame are
 * consecutive, in file order, and their segments and chunks follow one another inside the frame's ranges.  A scan
 * with several components (ncomp > 1) is interleaved: it codes the frame's mcus_x x mcus_y MCUs of bpm blocks, block
 * k of an MCU being component slot_comp[k] at (slot_dy[k], slot_dx[k]) inside it.  A one-component scan codes that
 * component's own blocks only, mcus_x = ceil(comp_w / 8) by mcus_y = ceil(comp_hgt / 8) in raster order (bpm 1), not
 * the MCU-padded plane.  restart counts MCUs (blocks of a one-component scan).  First scans (ah == 0: DC first,
 * AC first, sequential) store coefficients << al; refinement scans (ah != 0, al == ah - 1) add bit al.  dc[c] / ac[c]:
 * the Huffman tables in force at the scan's SOS for frame component c (those the scan uses).  8632 bytes. */
typedef struct acr_b200_jpeg_scan {
  int64_t coded_offset; /* entropy-coded segment: bytes [coded_offset, coded_offset + coded_len) of `coded` */
  int32_t coded_len;
  int32_t frame;        /* index of the file in `frames` */
  int32_t chunk_begin, n_chunks; /* ceil(coded_len / ACR_B200_JPEG_CHUNK) chunks, at least 1 */
  int32_t ncomp;        /* 1..3 components in the scan; 0: an unused descriptor (after every real one) */
  int32_t ss, se, ah, al; /* spectral selection and successive approximation (sequential: 0, 63, 0, 0) */
  int32_t restart;
  int32_t mcus_x, mcus_y, bpm, n_blocks; /* n_blocks = mcus_x * mcus_y * bpm */
  int8_t slot_comp[8], slot_dy[8], slot_dx[8];
  acr_b200_jpeg_huff dc[3], ac[3];
} acr_b200_jpeg_scan;

/* Workspace of acr_b200_jpeg_decode_scans for at most max_chunks chunks, max_blocks blocks and max_scans scans;
 * acr_b200_jpeg_coef_offset(max_chunks) is where its coefficient blocks are. */
size_t acr_b200_jpeg_scan_workspace_bytes(int64_t max_chunks, int64_t max_blocks, int64_t max_scans);

/* acr_b200_jpeg_decode for a batch that may hold multi-scan files (frames with n_scans > 0), described by the
 * max_scans descriptors at `scans` (device): the real ones first, sorted by frame, then unused ones (ncomp 0,
 * chunk_begin = the batch's chunk total, frame = INT32_MAX), so a CUDA graph replays with any mix of files.
 * Single-scan frames decode as in acr_b200_jpeg_decode, in the same launches.  The first scans of every file (DC
 * first, AC first, sequential) are decoded together with the same speculative chunks, one CTA per scan to
 * synchronise them; then one CTA per frame applies its refinement scans in file order (one thread walks each scan
 * to find every block's start from the blocks' nonzero masks, then the CTA decodes the blocks in parallel); then
 * the IDCT and colour conversion run over every frame.  A multi-scan frame's status is the OR of
 * its scans' (ACR_B200_JPEG_BAD_LENGTH also when a scan's blocks or EOB run pass its extent). */
int acr_b200_jpeg_decode_scans(const uint8_t* coded, int64_t coded_bytes, const acr_b200_jpeg_frame* frames, int n,
                               const acr_b200_jpeg_scan* scans, int64_t max_scans, int64_t max_chunks,
                               int64_t max_blocks, void* workspace, size_t workspace_bytes, uint8_t* out_bgr,
                               int64_t out_bytes, int32_t* status, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ACR_B200_H_ */
