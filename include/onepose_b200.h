/*
 * onepose_b200 -- C ABI of the H100-native GATsSPG 2D-3D matcher.
 *
 * The reference (zju3dv/OnePose) is pure Python and has no FFI; the boundary it
 * exposes for this path is `GATsSuperGlue.forward(data) -> (pred, conf_matrix)`
 * (reference src/models/GATsSPG_architectures/GATs_SuperGlue.py:179-241), reached
 * through `LitModelGATsSPG.forward` (src/models/GATsSPG_lightning_model.py:36-37)
 * from inference.py:146.  Each entry point below names the reference code it
 * replaces.  All signatures are plain C: pointers, sizes, a cudaStream_t passed
 * as void*.  No torch types.  Every function returns 0 on success or a negative
 * OPB_E_* code; opb_last_error() gives the message.  No exceptions cross the ABI.
 *
 * Pointer ownership: inputs are borrowed and never written; outputs are caller
 * allocated (device memory unless the name says _host).
 *
 * Streams and devices:
 *   - A handle (opb_matcher, opb_superpoint) owns one workspace and its objects.
 *     The library orders the calls of one handle across streams: a call on
 *     another stream than the handle's previous call first makes its stream wait
 *     for that call (cudaStreamWaitEvent; the host does not block).  Callers
 *     still order their own buffers (inputs, outputs) against their streams.
 *   - A handle's work runs on its own device (the `device` of its config); its
 *     inputs and outputs must live there.  Every handle entry point leaves the
 *     caller's current device as it found it.
 *   - The handle-free entry points (features3d producers, RANSAC-PnP, EPnP,
 *     gather, crop, detection, test hooks) run on the caller's current device
 *     and stream.  A call without a handle that fails -- these and the create
 *     functions -- leaves its message in a per-thread string that
 *     opb_last_error(NULL) and opb_sp_last_error(NULL) both return: the
 *     message of the last failed call on this thread that had no handle.
 *   - Calls on different handles may run concurrently, from different threads;
 *     one handle is used by one thread at a time.
 */
#ifndef ONEPOSE_B200_H_
#define ONEPOSE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OPB_OK 0
#define OPB_E_INVALID (-1)      /* bad argument / unsupported configuration        */
#define OPB_E_CUDA (-2)         /* CUDA runtime / driver error                      */
#define OPB_E_STATE (-3)        /* call order violated (weights / object missing)   */
#define OPB_E_RANGE (-4)        /* activation left the fp16-split operand range     */
#define OPB_E_NOT_IMPLEMENTED (-5)

typedef struct opb_matcher opb_matcher; /* opaque */

/* Hyper-parameters = the `hparams` mapping of GATsSuperGlue.__init__
 * (GATs_SuperGlue.py:145-177; released values configs/experiment/train_GATsSPG.yaml:44-60). */
typedef struct opb_config {
  int32_t descriptor_dim;        /* 256 (only value supported)                         */
  int32_t num_heads;             /* 4   (GATs_SuperGlue.py:43)                          */
  float scale_factor;            /* 0.07 (GATs_SuperGlue.py:217); >= 2 log2(e) / 126    */
  float match_threshold;         /* 0.2  (GATs_SuperGlue.py:227)                        */
  int32_t include_self;          /* GATs.py:48                                          */
  int32_t additional;            /* GATs.py:61                                          */
  int32_t with_linear_transform; /* GATs.py:56-57,64-65                                 */
  int32_t device;                /* CUDA device ordinal                                 */
} opb_config;

/* Replaces GATsSuperGlue.__init__ (GATs_SuperGlue.py:145-177). */
int opb_create(const opb_config* cfg, opb_matcher** out);
void opb_destroy(opb_matcher* m);
const char* opb_last_error(const opb_matcher* m); /* m may be NULL: last failed call without a handle on this thread */

/* Replaces nn.Module.load_state_dict for the keys of GATs_SuperGlue.py (SURVEY 2.1):
 * `name` is the reference state-dict key ("gnn.layers.1.attn.proj.0.weight", ...),
 * `data` a HOST fp32 array in the reference's own layout.  Dead parameters
 * (kenc_*, bin_score) are accepted and ignored.  opb_finalize_weights() packs
 * (head permutation, merge->mlp.0 folding, W.a folding, fp16 hi/lo split) and uploads. */
int opb_load_weight(opb_matcher* m, const char* name, const float* data, size_t n_elems);
int opb_finalize_weights(opb_matcher* m);

/* Per-object constants = the tensors inference.py:113-130 builds once per sequence
 * and pack_data (inference.py:80-94) re-uploads every frame:
 *   desc3d_db  device fp32 [256, M]    (descriptors3d_db, channel-first)
 *   desc2d_db  device fp32 [256, M*L]  (descriptors2d_db, column i*L+j = leaf j of point i; GATs.py:46) */
int opb_set_object(opb_matcher* m, const float* desc3d_db, const float* desc2d_db,
                   int32_t M, int32_t L, void* stream);

/* Size the chunk workspace for calls of up to `frames` frames of up to N query points each (SURVEY 8b: no allocation on the
 * hot path beyond a workspace sized with the object).  Optional: opb_forward grows the workspace itself on first use / when a
 * call exceeds what was reserved (a one-time cudaMalloc + device synchronisation). */
int opb_reserve_workspace(opb_matcher* m, int32_t frames, int32_t N);

/* Replaces GATsSuperGlue.forward (GATs_SuperGlue.py:179-241) for B query frames of
 * the current object.  desc2d_query: device fp32 [B, 256, N] (channel-first, as in
 * the reference).  n2d_lengths: device int32 [B] = valid query points of each frame (SuperPoint yields a different count per
 * frame, src/sfm/extract_features.py:19-24; columns >= n2d_lengths[b] of frame b are ignored) or NULL = N everywhere.
 * Outputs (device): matches0 int64 [B,N], matches1 int64 [B,M], mscores0 fp32 [B,N], mscores1 fp32 [B,M]; conf fp32 [B,N,M]
 * or NULL to skip materialising the confidence matrix.  Entries of a frame beyond its length are -1 / 0.  A length of 0 is
 * valid: that frame matches nothing (-1 / 0 everywhere, conf rows 0), its 3D points receive no cross-attention message, and
 * the other frames of the call are unaffected.
 * Asynchronous on `stream`; no host synchronisation. */
int opb_forward(opb_matcher* m, const float* desc2d_query, const int32_t* n2d_lengths, int32_t B, int32_t N,
                int64_t* matches0, int64_t* matches1, float* mscores0, float* mscores1,
                float* conf, void* stream);

/* Several objects on one handle.  opb_add_object uploads an object's constants (arguments as opb_set_object) and returns its
 * id in *object_id; its GNN prologue runs on its first use, once.  The registration is independent of opb_set_object's
 * current object.  opb_finalize_weights keeps registered objects: their leaf logits and prologue are recomputed under the new
 * weights on their next use.  opb_remove_object frees an object after the work in flight (it synchronises the device). */
int opb_add_object(opb_matcher* m, const float* desc3d_db, const float* desc2d_db, int32_t M, int32_t L, void* stream,
                   int32_t* object_id);
int opb_remove_object(opb_matcher* m, int32_t object_id);

/* opb_forward for frames of different objects in one call: frame b matches against object object_ids_host[b] (HOST int32
 * [B], registered ids; every object of a call has the same L, M may differ).  desc2d_query / n2d_lengths as in opb_forward.
 * Outputs (device): matches0 int64 [B,N], mscores0 fp32 [B,N], matches1 int64 [B,M_out], mscores1 fp32 [B,M_out], conf fp32
 * [B,N,M_out] or NULL; M_out >= the largest M of the call.  Columns >= M_b of frame b (its object's M) are -1 in matches1 and
 * 0 in mscores1 and conf.  A frame's results do not depend on the other frames of the call.  OPB_E_INVALID for an unknown
 * id, objects with different L, M_out too small, B <= 0 or N <= 0.  The range guard reports as for opb_forward.
 * Asynchronous on `stream`; no host synchronisation. */
int opb_forward_objects(opb_matcher* m, const int32_t* object_ids_host, const float* desc2d_query, const int32_t* n2d_lengths,
                        int32_t B, int32_t N, int32_t M_out, int64_t* matches0, int64_t* matches1, float* mscores0, float* mscores1,
                        float* conf, void* stream);

/* Same call with HOST buffers (pinned or pageable): H2D of the query descriptors (and lengths, may be NULL),
 * forward, D2H of matches/scores; returns after the stream has been synchronised.  The confidence matrix is
 * materialised on the device if conf_host is non-NULL (then also copied back) or materialize_conf != 0
 * (the reference always computes it; inference.py:146 discards it).  This is the end-to-end leg bench.py times. */
int opb_forward_host(opb_matcher* m, const float* desc2d_query_host, const int32_t* n2d_lengths_host, int32_t B, int32_t N,
                     int64_t* matches0_host, int64_t* matches1_host, float* mscores0_host,
                     float* mscores1_host, float* conf_host, int32_t materialize_conf, void* stream);

/* Range guard of the fp16-split operand format (|x| < 1023 per plane element).  A call that produced an activation outside the
 * range (or a NaN) reports "no match" (-1 / 0) for every point on the device, and the error is delivered to the host lazily:
 *   opb_poll_range   never blocks: OPB_E_RANGE if a finished earlier call raised the flag, OPB_OK otherwise (also while
 *                    the last call is still running);
 *   opb_check_range  waits for the handle's last call and reports.  opb_forward_host calls it itself.
 * Reporting clears the flag; the clearing is ordered before the handle's next call, on whatever stream. */
int opb_check_range(opb_matcher* m, void* stream);
int opb_poll_range(opb_matcher* m);

/* Number of kernels opb_forward launched in its last call (bench.py "gpu_launches"). */
int opb_last_launch_count(const opb_matcher* m);

/* Measurement hook for bench.py: with profiling on, every launch of opb_forward is followed by a CUDA event on the launch
 * stream.  opb_get_profile() synchronises and returns the summed GEMM time, the ALGORITHMIC FLOPs those launches performed
 * (2*valid_rows*n_out*K, each logical MMA counted once although it executes as 3 fp16 passes), their count, and the time of the
 * whole forward (first to last kernel).  Profiling perturbs timing slightly: never on in timed runs. */
int opb_set_profiling(opb_matcher* m, int32_t enable);
int opb_get_profile(opb_matcher* m, double* gemm_ms, double* gemm_flops, int32_t* gemm_launches, double* total_ms);
/* Same for the launches whose profile name starts with `prefix` ("gemm epi1 " = the mlp.0 GEMM, "kv_state", ...). */
int opb_get_profile_entry(opb_matcher* m, const char* prefix, double* ms, double* flops, int32_t* launches);

/* GNN layers 0 (GATs) and the 3D side of layer 1 (self) depend only on the per-object constants; by default they
 * are evaluated once per opb_forward call and shared by its frames.  enable = 0 evaluates them per frame like the
 * reference does (same results up to fp32 rounding; used by the tests). */
int opb_set_hoist(opb_matcher* m, int32_t enable);

/* Frames processed together through the GNN (workspace-size knob); 0 = default (32).  At most 64: larger values return
 * OPB_E_INVALID and leave the setting unchanged. */
int opb_set_chunk_frames(opb_matcher* m, int32_t frames);

/* ---- adjacent producers: the per-object feature files the path consumes (SURVEY 8f N2) ---- */
/* mean_descriptors (reference src/sfm/postprocess/feature_process.py:297-305, fp64): seg_len device int64 [M] track lengths,
 * out device f64 [M, D] = np.mean of each track's rows, bit-identical, in the summation order numpy uses for the layout given
 * (its reduction loop runs along the axis with the smaller stride).  Both sums start from +0.0; a zero-length track gives NaN.
 * opb_segmented_mean_f64: desc device f64 [sum(seg_len), D] row-major (numpy on C-ordered input, D > 1): the rows are added
 * in order, one running sum per channel. */
int opb_segmented_mean_f64(const double* desc, const int64_t* seg_len, int32_t M, int32_t D,
                           double* out, void* stream);
/* opb_segmented_mean_channels_f64: desc device f64 [D, sum(seg_len)], each channel's observations contiguous (numpy on
 * F-ordered input such as the transpose of channel-first features, or D = 1): each channel's track is summed pairwise. */
int opb_segmented_mean_channels_f64(const double* desc, const int64_t* seg_len, int32_t M, int32_t D, double* out, void* stream);
/* mean_scores (feature_process.py:308-317, fp64): scores device f64 [sum(seg_len)] -> out device f64 [M]; the D = 1 case of
 * opb_segmented_mean_channels_f64 (pairwise, as numpy sums a contiguous run). */
int opb_segmented_mean_scores_f64(const double* scores, const int64_t* seg_len, int32_t M, double* out, void* stream);
/* Column gather of pad_features3d_random / build_features3d_leaves (reference src/utils/data_utils.py:143-205):
 * desc device fp32 [dim, n_src] (channel-first), scores device fp32 [n_src] (may be NULL), idx device int64 [n_idx] = source
 * column of each output column (n_src = the all-ones / zero-score dustbin; NULL = identity) -> desc_out [dim, n_out],
 * scores_out [n_out]; output columns >= n_idx are all-ones / zero padding.  dim <= 65535; n_out = 0 writes nothing. */
int opb_gather_features3d(const float* desc, const float* scores, int32_t dim, int64_t n_src, const int64_t* idx, int64_t n_idx,
                          float* desc_out, float* scores_out, int64_t n_out, void* stream);

/* ---- adjacent consumer: object pose from the matched correspondences (SURVEY 8f N3) ----
 * Replaces the per-frame cv2.solvePnPRansac(..., reprojectionError=5, iterationsCount=10000, flags=SOLVEPNP_EPNP) of
 * ransac_PnP (reference src/utils/eval_utils.py:18-42) for B frames in one call, on the device:
 *   K          device f64 [B, 9]   row-major camera matrices
 *   pts2d      device f64 [total, 2], pts3d device f64 [total, 3]  matched key points of all frames, concatenated
 *   offsets    device int32 [B+1]  frame b owns correspondences [offsets[b], offsets[b+1]); offsets[0] may be above 0, and
 *              inlier_mask rows outside every frame are never written
 *   hypotheses minimal samples per frame (P3P), 1 .. 65535 * 128; reproj_error in pixels, > 0 (inf allowed; 0, negative and
 *              NaN are refused, where OpenCV squares a negative threshold); seed of the sample generator
 *              (results are a deterministic function of it)
 *   workspace  device f64 [B * hypotheses * 13]: one record of 13 doubles per frame and hypothesis, frame-major
 *              (record b * hypotheses + h): the inlier count of the hypothesis's best P3P pose, then that pose's R (9,
 *              row-major) and t (3).  A record with count 0 (frame with fewer than 4 correspondences, or no P3P solution)
 *              leaves its pose unwritten.  Sample h of frame b is three distinct indices drawn from
 *              splitmix64(seed ^ (b << 40) ^ h) and its successors.
 * Outputs (device): pose f64 [B, 12] = row-major [R | t] (world -> camera), inlier_mask int32 [total], n_inliers int32 [B].
 * A frame with fewer than 4 correspondences or no model gets the identity pose and no inliers (the reference's cv2.error
 * branch).  Inlier: in front of the camera and squared reprojection error < reproj_error^2, in fp64; a pair with a NaN or an
 * infinity is never one, and a sample holding one has no model.  A refinement that ends with fewer than 4 inliers (a
 * threshold that admits gross outliers can drag the pose off the object) gives way to the winning hypothesis's pose.  K:
 * only fx = K[0], fy = K[4], cx = K[2], cy = K[5] are read (skew and the last row are ignored, as OpenCV's EPnP and
 * projectPoints ignore them).  Parity with the reference is on the pose (cm / degree), not on bits: OpenCV draws its own
 * samples. */
int opb_ransac_pnp(const double* K, const double* pts2d, const double* pts3d, const int32_t* offsets, int32_t B, int32_t hypotheses,
                   double reproj_error, uint64_t seed, double* workspace, double* pose_out, int32_t* inlier_mask, int32_t* n_inliers,
                   void* stream);
/* EPnP (Lepetit, Moreno-Noguer, Fua, IJCV 2009) on all correspondences of each frame: cv2.solvePnP(..., flags=SOLVEPNP_EPNP)
 * for B frames, one block per frame, fp64, fixed-order reductions (deterministic).  K, pts2d, pts3d, offsets as for
 * opb_ransac_pnp (used as given, no rounding).  Outputs (device): pose f64 [B, 12] row-major [R | t], status int32 [B] = 1 for
 * a pose, 0 with the identity pose for a frame with fewer than 4 correspondences or a non-finite result (coincident or
 * collinear points, or no candidate with solvable betas).  Control points: the centroid and the principal axes scaled by
 * sqrt(lambda / n), each axis with its largest-magnitude component positive (on noisy data the answer depends on these
 * signs; OpenCV takes its SVD's, so its pose can differ from this one by the noise's effect); for a planar set (third
 * eigenvalue below 1e-10 of the first) the third control point sits at the first axis's length along the normal, and the
 * null vector with the least weight on its columns comes first.  The null space of M^T M by Jacobi rotations; candidates for
 * N = 1, 2, 3 null vectors, each refined by 5 Gauss-Newton steps on the four betas; R, t by Horn's quaternion; the lowest
 * mean reprojection error wins, the first candidate on ties. */
int opb_epnp(const double* K, const double* pts2d, const double* pts3d, const int32_t* offsets, int32_t B, double* pose_out,
             int32_t* status, void* stream);
/* EPnP-RANSAC: the reference's cv2.solvePnPRansac(..., flags=SOLVEPNP_EPNP) for B frames; same arguments, workspace records and
 * outputs as opb_ransac_pnp, no host synchronisation.
 *   inputs      every correspondence is rounded to fp32 first (as OpenCV converts its inputs); K is used as given;
 *   hypotheses  sample h of frame b: r = splitmix64(seed ^ (b << 40) ^ h); index k (k = 0..4) is the next state modulo
 *               n - k, increased by one for every earlier index it reaches (taken in ascending order), so the five are
 *               distinct; EPnP on them (the routine of opb_epnp, one thread).  A frame of exactly 4 correspondences solves
 *               P3P on correspondences 0-2 and keeps the solution that reprojects 3 best: OpenCV also fits a 4-point model
 *               there (it returns a pose with 4 inliers where no 5-point sample exists: tests/golden/make_epnp.py);
 *   count       inliers over all n by OpenCV's rule: squared reprojection error <= reproj_error^2, in fp64, with no depth
 *               test (points behind the camera that project close enough count); a non-finite pose counts 0, and a
 *               non-finite error (a pair with a NaN or an infinity) is never an inlier, not even at reproj_error = inf;
 *   selection   most inliers, lowest index on ties (the arg-max of opb_ransac_pnp);
 *   refit       EPnP (the block routine of opb_epnp) on the winning sample's inlier set, which is the reported inlier_mask.
 * Fewer than 4 correspondences, or a best count below 4, gives the identity pose and no inliers.  OpenCV raises or returns
 * false there instead, and the reference's ransac_PnP turns that into the same identity pose and empty inlier list.  OpenCV
 * draws its samples from its own serial, adaptive sequence, so parity is on the pose, not on bits. */
int opb_ransac_epnp(const double* K, const double* pts2d, const double* pts3d, const int32_t* offsets, int32_t B, int32_t hypotheses,
                    double reproj_error, uint64_t seed, double* workspace, double* pose_out, int32_t* inlier_mask, int32_t* n_inliers,
                    void* stream);
/* EPnP-RANSAC as OpenCV runs it: cv2.solvePnPRansac(..., iterationsCount=hypotheses, confidence, flags=SOLVEPNP_EPNP) for B
 * frames, with OpenCV's sample sequence and stopping rule; no host synchronisation.  Arguments as opb_ransac_epnp without the
 * seed (OpenCV's generator starts from the same state on every call), plus:
 *   hypotheses  1 .. 65535 * 128 (OpenCV runs iterationsCount = 0 as one iteration; 0 is refused here)
 *   confidence  0 .. 1 (OpenCV's run() asserts 0 < confidence < 1; 0 and 1 follow RANSACUpdateNumIters' clamped formula:
 *               0 stops after the first winning sample; 1 lowers the budget to at most
 *               cvRound(log(DBL_MIN) / log(1 - (1 - outlier ratio)^5)), e.g. about 8700 at 40 % outliers)
 *   workspace   device f64 [B * (hypotheses * 13 + 16)]
 *   iterations  device int32 [B] out: the iter at which OpenCV's loop exits (0 for frames of fewer than 6 pairs)
 * Per frame, as RANSACPointSetRegistrator::run (calib3d/src/ptsetreg.cpp) with PnPRansacCallback:
 *   samples     cv::RNG from state 2^64 - 1: state = (uint32)state * 4164903690 + (state >> 32), index = (uint32)state % n;
 *               five per sample, an index equal to an earlier one of the same sample drawn again; sample i of a frame is the
 *               i-th subset OpenCV draws for its n;
 *   model       EPnP on the five fp32-rounded pairs (the routine of opb_ransac_epnp); no finite pose = no model;
 *   count       OpenCV's fp32 error: the projection in fp64 rounded to fp32, the squared distance in fp32, <= the bound
 *               fp32(fp32(reproj_error)^2): solvePnPRansac takes a float threshold and findInliers squares it in double
 *               and rounds to float.  This is not (float)(reproj_error^2), which is one ulp off for about half of all
 *               thresholds (5.3, 0.7, ...).  A non-finite error is never an inlier (OpenCV counts an infinite one at
 *               reproj_error = inf);
 *   loop        sample i wins when its count > max(best, 4) (the earliest wins a tie); each win lowers the budget to
 *               RANSACUpdateNumIters(confidence, outlier ratio, 5, budget); the loop exits at iter >= budget;
 *   result      the winner's inlier set is inlier_mask (n_inliers its count), the pose EPnP on it.  No winner: the identity
 *               pose and no inliers.  Frames of 4 or 5 pairs are solved once from all of them, every pair an inlier and no
 *               refit, as solvePnPRansac does when npoints == model_points: 4 pairs by the 4-pair model of opb_ransac_epnp
 *               (P3P on 0-2, the solution that best reprojects 3; solvePnP(P3P)), 5 by the per-thread EPnP on all five
 *               (solvePnP(EPNP)).  Fewer than 4 pairs get the identity pose.
 * Samples are evaluated in waves of W per frame (W chosen from B to fill the device); a frame skips every wave after the one
 * its loop ends in, so a call costs the waves of its slowest frame, at most ceil(hypotheses / W).  Results past the exit are
 * discarded, so the outputs do not depend on W. */
int opb_ransac_epnp_cv(const double* K, const double* pts2d, const double* pts3d, const int32_t* offsets, int32_t B, int32_t hypotheses,
                       double reproj_error, double confidence, double* workspace, double* pose_out, int32_t* inlier_mask,
                       int32_t* n_inliers, int32_t* iterations, void* stream);
/* Test hooks of opb_ransac_epnp_cv.  opb_debug_set_cv_wave: W for later calls (0 = chosen from B).  opb_debug_set_cv_trace:
 * device buffers later calls fill (NULL to stop): samples int32 [B][capacity][5] and counts int32 [B][capacity] for every
 * sample i < capacity the loop evaluates (count -1: no model), winner int32 [B] (-1: none).  opb_debug_cv_subsets: the first
 * count samples of a frame of n >= 5 pairs into out int32 [count][5], by the device's generator, drawn `chunk` at a time
 * (as the waves draw them). */
int opb_debug_set_cv_wave(int32_t wave);
int opb_debug_set_cv_trace(int32_t* samples, int32_t* counts, int32_t* winner, int32_t capacity);
int opb_debug_cv_subsets(int32_t n, int32_t count, int32_t chunk, int32_t* out, void* stream);
/* Matched 2D-3D pairs of B frames in the layout opb_ransac_pnp reads; replaces inference.py:147-152 / eval_utils.py:72-77
 * (valid = matches0 > -1; mkpts2d = kpts2d[valid]; mkpts3d = kpts3d[matches0[valid]]; mconf = scores0[valid]).
 *   matches0     device int64 [B, N]  (opb_forward's output; an entry outside [0, M) is not a match)
 *   mscores0     device fp32  [B, N]  or NULL (then mconf must be NULL)
 *   keypoints2d  device fp32  [B, N, 2]  (x, y; opb_sp_forward's keypoints with cap = N; rows of unmatched entries are never read)
 *   keypoints3d  device fp32  [M, 3]
 * Outputs (device, capacity B*N): pts2d f64 [B*N, 2], pts3d f64 [B*N, 3], mconf fp32 [B*N] or NULL,
 * query_index int32 [B*N] or NULL (= n of each pair), offsets int32 [B+1] (frame b owns [offsets[b], offsets[b+1])).
 * Pairs are frame-major and, within a frame, in ascending n: numpy boolean-mask order.  The values are exact (fp32 -> f64
 * conversions, as numpy's astype(np.float64)).  Three launches, deterministic, no host synchronisation.  B*N < 2^31;
 * matches0 / keypoints2d / pts2d / pts3d may be NULL when N = 0 (then offsets = 0). */
int opb_gather_matches(const int64_t* matches0, const float* mscores0, const float* keypoints2d, const float* keypoints3d,
                       int32_t B, int32_t N, int32_t M, double* pts2d, double* pts3d, float* mconf, int32_t* query_index,
                       int32_t* offsets, void* stream);
/* The same for frames of different objects (opb_forward_objects' output):
 *   keypoints3d  device fp32 [sum M, 3]  the objects' 3D key points, concatenated
 *   kp3_first    device int32 [B]        first row of frame b's object in keypoints3d
 *   kp3_count    device int32 [B]        its M: an entry m of frame b is a match iff 0 <= m < kp3_count[b]
 * Other arguments, outputs and order as opb_gather_matches, which is this call with kp3_first = 0 and kp3_count = M. */
int opb_gather_matches_objects(const int64_t* matches0, const float* mscores0, const float* keypoints2d, const float* keypoints3d,
                               const int32_t* kp3_first, const int32_t* kp3_count, int32_t B, int32_t N, double* pts2d, double* pts3d,
                               float* mconf, int32_t* query_index, int32_t* offsets, void* stream);

/* ---- colour camera frames to the grey frames every frame consumer below takes (csrc/frames.cu) ----
 * The reference reads its frames as cv2.imread(path, cv2.IMREAD_GRAYSCALE) of the colour PNGs parse_scanned_data.py writes
 * (NormalizedDataset, src/datasets/normalized_dataset.py:25-34; read_gray_scale, src/utils/data_utils.py:275-276;
 * local_feature_2D_detector.py:12, :155, :173).  opb_grey_frames makes those grey pixels from colour pixels in device memory
 * -- a camera's or cv2.VideoCapture's frames -- and optionally NormalizedDataset's `image / 255.`.  On the caller's current
 * device and stream; asynchronous, no host synchronisation, no allocation.
 *   frames            device uint8 [F, H, W, C]  8-bit pixels, C = 3 or 4 by `order`; frame f starts at frames + f * frame_pitch,
 *                     its row y at + y * row_pitch (bytes; row_pitch >= W * C; frame_pitch 0, one frame for all F, or
 *                     >= H * row_pitch).  F <= 65535, H, W <= 32767 (the crop's bounds)
 *   order             OPB_ORDER_BGR, _RGB, _BGRA or _RGBA: the channels of a pixel in memory order; alpha is ignored
 *   grey              device uint8 [F, H, W] out, with its own pitches: grey_row_pitch >= W, grey_frame_pitch >= H * grey_row_pitch
 *   image             device fp32 [F, 1, H, W] out (dense), or NULL: grey / 255 as a float32 division, numpy's `image / 255.`
 * grey = (9797 * R + 19234 * G + 3737 * B) >> 15, OpenCV 4.13's IMREAD_GRAYSCALE of a colour 8-bit PNG, bit for bit on every
 * colour (the model is tests/grey_reference.py).  It is not cv2.cvtColor(COLOR_BGR2GRAY), which differs by one level on half
 * of the colours.  The outputs must not overlap the frames or each other. */
enum { OPB_ORDER_BGR = 0, OPB_ORDER_RGB = 1, OPB_ORDER_BGRA = 2, OPB_ORDER_RGBA = 3 };
int opb_grey_frames(const uint8_t* frames, int64_t frame_pitch, int64_t row_pitch, int32_t F, int32_t H, int32_t W, int32_t order, uint8_t* grey,
                    int64_t grey_frame_pitch, int64_t grey_row_pitch, float* image, void* stream);

/* ---- between one frame's pose and the next frame's extractor input: the pose-guided crop ----
 * The reference's live loop (inference_demo.py:193-247) crops every frame after the first around the object's box under the
 * previous pose: previous_pose_detect (src/local_feature_2D_detector/local_feature_2D_detector.py:232-259), host numpy +
 * cv2.warpAffine.  The three calls below do it for B frames on the caller's current device and stream: device pointers,
 * asynchronous, no host synchronisation, no allocation; OPB_E_INVALID for null or non-positive arguments.  B <= 65535.
 *
 * Box of the object's 3D bounding-box corners under a pose; replaces reproj (src/utils/vis_utils.py:209-236) and
 * local_feature_2D_detector.py:246-249 (min / max over the corners, astype(np.int32)).
 *   K        device f64 [B, 9]             row-major camera matrices
 *   pose     device f64 [B, 12]            row-major [R | t], the pose_out layout of opb_ransac_*
 *   corners  device f64 [B, n_corners, 3]  (8 in the reference; any n_corners > 0)
 *   proj     device f64 [B, n_corners, 2]  out, or NULL: the projections, reproj's result
 *   box      device int32 [B, 4]           out: [x0, y0, x1, y1]
 * Per frame, in fp64 with every product and sum rounded on its own and summed in index order: (K @ pose) @ [X; 1], the
 * division by the third row, min / max, then C truncation towards zero (numpy's cast).  A corner behind the camera projects
 * as it does in numpy.  A non-finite extreme or one outside int32, where numpy's cast is undefined, gives the empty box
 * [0, 0, 0, 0], which opb_crop_resize rejects. */
int opb_boxes_from_poses(const double* K, const double* pose, const double* corners, int32_t B, int32_t n_corners, double* proj,
                         int32_t* box, void* stream);
/* crop_img_by_bbox (local_feature_2D_detector.py:160-186) and the `/ 255` of :255-257: the two chained get_image_crop_resize and
 * get_K_crop_resize calls (src/utils/data_utils.py:233-272), box -> an image of the box's own size -> crop_size x crop_size.
 *   frames      device uint8 [B, H, W]  full grey camera frames; frame b starts at frames + b * frame_pitch, its row y at
 *               + y * row_pitch (bytes; row_pitch >= W); H, W <= 32767
 *   box         device int32 [B, 4]     [x0, y0, x1, y1]
 *   K           device f64 [B, 9]
 *   crop_size   S > 0, S % 8 == 0 (the extractor's condition; 512 in the reference)
 *   image       device fp32 [B, 1, S, S] out: the `images` argument of opb_sp_forward
 *   K_crop      device f64 [B, 9] out:   T2_homo @ [ (T1_homo @ [K | 0])[:3, :3] | 0 ], fp64, products summed in index order
 *   trans       device f64 [B, 2, 6] out: T1 and T2, row-major 2x3 (T2 . T1 maps a frame position into the crop)
 *   status      device int32 [B] out:    1, or 0 for a rejected box
 * A box is rejected when x1 <= x0 or y1 <= y0 (the reference raises inside cv2 there), when a side exceeds 32767 or a
 * coordinate 2^20 in magnitude (cv2 addresses source pixels by int16 and positions in 22.10 fixed point): status 0, a zero
 * image, zero transforms and K_crop = K.  A zero image yields no key points, hence the identity pose and 0 inliers from
 * opb_ransac_*: the failure reaches the caller through n_inliers, the signal inference_demo.py:206 uses.
 * Arithmetic (bit-exact against OpenCV 4.13; the model is tests/crop_reference.py):
 *   transforms  get_affine_transform (data_utils.py:24-57, rot = 0): three float32 point pairs -- the centre, the point half
 *               the WIDTH above it, get_3rd_point of the two -- then cv2.getAffineTransform's 6x6 system solved in fp64 by LU
 *               with partial pivoting in OpenCV's elimination order, no fused multiply-add.  Both axes scale by dst_w / src_w:
 *               the reference's crop is not an anisotropic resize.
 *   pixels      cv2.warpAffine(INTER_LINEAR, constant border 0) on 8-bit data: the matrix inverted in fp64 as warpAffine does,
 *               source positions rint((M . (x, y, 1)) * 1024) (round half to even) reduced to 1/32, the pixel index
 *               saturated to int16, four int16 weights rint(w * 32768) per 1/32 x 1/32 fraction, pixel = (sum + 16384) >> 15.
 *               Each output pixel evaluates the 4 first-stage pixels it needs (rounded to uint8, zero outside the first-stage
 *               image) from 16 frame reads; no intermediate image.  The result is the uint8 value / 255 in fp32 (numpy's). */
int opb_crop_resize(const uint8_t* frames, int64_t frame_pitch, int64_t row_pitch, int32_t B, int32_t H, int32_t W, const int32_t* box,
                    const double* K, int32_t crop_size, float* image, double* K_crop, double* trans, int32_t* status, void* stream);
/* opb_crop_resize for B crops of n_frames frames (several boxes per frame): crop b reads frame frame_index[b].
 *   frames        device uint8 [n_frames, H, W] with the pitches of opb_crop_resize
 *   frame_index   device int32 [B]
 *   B <= 65535; box, K, crop_size, image, K_crop, trans, status as in opb_crop_resize, per crop.
 * Crop b equals, bit for bit, opb_crop_resize's crop b of the gathered frames frames[frame_index[b]].  An index outside
 * [0, n_frames) is rejected as a rejected box is: status 0, a zero image, zero transforms and K_crop = K. */
int opb_crop_resize_indexed(const uint8_t* frames, int64_t frame_pitch, int64_t row_pitch, int32_t n_frames, int32_t H, int32_t W,
                            const int32_t* frame_index, int32_t B, const int32_t* box, const double* K, int32_t crop_size, float* image,
                            double* K_crop, double* trans, int32_t* status, void* stream);
/* One get_image_crop_resize / get_K_crop_resize (data_utils.py:233-272): box -> [out_h, out_w] by one warp -- the pixel and
 * transform routines opb_crop_resize runs twice.  frames, pitches, box as there; out_h, out_w <= 32767.
 *   out     device uint8 [B, out_h, out_w] out: cv2.warpAffine's image.  frames and out may both be NULL: transforms only
 *   trans   device f64 [B, 6] out: trans_crop, row-major 2x3
 *   K, K_crop  device f64 [B, 9] in / out: trans_crop_homo @ K, or both NULL
 * A rejected box (as for opb_crop_resize) gives a zero image, a zero transform and K_crop = K. */
int opb_warp_crop_u8(const uint8_t* frames, int64_t frame_pitch, int64_t row_pitch, int32_t B, int32_t H, int32_t W, const int32_t* box,
                     const double* K, int32_t out_h, int32_t out_w, uint8_t* out, double* trans, double* K_crop, void* stream);
/* opb_crop_resize's two warps on colour frames, into uint8: the crops parse_scanned_data.py's parse_video writes to color/
 * (:151-159, cv2.warpAffine of the BGR frame, then of its first-stage crop).
 *   frames        device uint8 [n_frames, H, W, C], C = 3 or 4, packed pixels; frame f starts at frames + f * frame_pitch, its
 *                 row y at + y * row_pitch (bytes; row_pitch >= W * C, frame_pitch >= 0)
 *   frame_index   device int32 [B], or NULL: crop b reads frame frame_index[b] (an index outside [0, n_frames) is rejected as a
 *                 rejected box is), or frame b, with n_frames == B
 *   image         device uint8 [B, S, S, C] out: every channel warped as cv2.warpAffine warps a C-channel 8-bit image
 *   box, K, crop_size, K_crop, trans, status as in opb_crop_resize, per crop.
 * Channel c of crop b equals, bit for bit, opb_crop_resize's pixels (times 255) of plane c of the same frame: cv2 warps every
 * channel with the grey warp's positions and weights.  A rejected box gives a zero crop, zero transforms and K_crop = K. */
int opb_crop_resize_colour(const uint8_t* frames, int64_t frame_pitch, int64_t row_pitch, int32_t n_frames, int32_t H, int32_t W, int32_t C,
                           const int32_t* frame_index, int32_t B, const int32_t* box, const double* K, int32_t crop_size, uint8_t* image,
                           double* K_crop, double* trans, int32_t* status, void* stream);

/* ---- an annotated scan's poses, boxes and crop geometry (csrc/scan.cu) ----
 * parse_scanned_data.py's data_process_anno (:184-240) and parse_video (:129-181) turn an ARKit scan -- ARposes.txt, Box.txt,
 * Frames.txt and the video -- into the object poses, boxes and 512 x 512 colour crops inference.py evaluates against.  The two
 * calls below, with opb_crop_resize_colour between them, do its arithmetic on the caller's current device and stream: device
 * pointers, asynchronous, no host synchronisation, no allocation.  fp64 with every product and sum rounded on its own in numpy's
 * index order; the model is tests/scan_reference.py.
 *
 * data_process_anno's loop (downsample_rate = 1) over n_rows ARposes rows, in one launch:
 *   K          device f64 [9]              the averaged intrinsics (K_homo = [K | 0])
 *   arposes    device f64 [n_rows, 8]      (timestamp, x, y, z, qw, qx, qy, qz) per row, comment and blank lines removed
 *   T_ow       device f64 [16]             Box.txt's object-to-world transform, row-major
 *   corners    device f64 [n_corners, 3]   the object's box corners (8 from Box.txt); n_corners <= 1024
 *   pose       device f64 [n_out, 16] out  T_oc of the kept rows in order, row-major; zeros in slots past the kept count
 *   proj       device f64 [n_out, n_corners, 2] out, or NULL: reproj(K_homo, T_oc, corners) of the kept rows; zeros past them
 *   box        device int32 [n_out, 4] out [x0, y0, x1, y1], the projection's min / max truncated towards zero (parse_video's
 *                                          astype(int)); [0, 0, 0, 0] past the kept rows, or for a NaN extreme
 *   row        device int32 [n_out] out, or NULL: the ARposes row of each slot; -1 past the kept rows
 *   keep       device int32 [n_rows] out, or NULL: 1 for a kept row, 0 for a skipped one
 *   count      device int32 [1] out: the number of kept rows
 * Per row: R = quat2mat(q) (transforms3d's non-normalising formula: s = 2 / |q|^2, the identity for |q|^2 < float64 eps),
 * R @ diag(1, -1, -1), T_cw = [R p; 0 1], T_oc = inv(T_cw) @ T_ow, the projection of the corners and its min / max.  A row is
 * skipped when x0 < -1000, y0 < -1000, x1 > 3000 or y1 > 3000 (a NaN extreme fails these tests and is kept, as in numpy).  A
 * skipped row does not advance the reference's index, and parse_video stops at the first index without a box file, so video
 * frame i pairs with the i-th kept row and frames past the kept count get nothing: slot i of the outputs is frame i's. */
int opb_scan_poses(const double* K, const double* arposes, int32_t n_rows, const double* T_ow, const double* corners, int32_t n_corners,
                   int32_t n_out, double* pose, double* proj, int32_t* box, int32_t* row, int32_t* keep, int32_t* count, void* stream);
/* parse_video's crop-to-frame transform and box in crop coordinates for F frames, one thread per frame:
 *   trans      device f64 [F, 2, 6]         T1 and T2 of opb_crop_resize_colour
 *   K_crop     device f64 [F, 9]            its K_crop
 *   pose       device f64 [F, 16]           T_oc (opb_scan_poses' pose)
 *   corners    device f64 [n_corners, 3]    n_corners <= 1024
 *   status     device int32 [F]             opb_crop_resize_colour's status
 *   M          device f64 [F, 9] out        inv(T2_homo @ T1_homo), the crop-to-frame transform written to M/
 *   box_crop   device f64 [F, 4] out        min / max of reproj(K_crop_homo, T_oc, corners), not truncated (bbox/)
 * Both are zero for a frame of status 0. */
int opb_scan_crop_geometry(const double* trans, const double* K_crop, const double* pose, const double* corners, int32_t n_corners,
                           const int32_t* status, int32_t F, double* M, double* box_crop, void* stream);

/* ---- the first frame, and every frame after a lost pose: detection by 2D-2D matching against reference views ----
 * LocalFeatureObjectDetector.detect (local_feature_2D_detector.py:76-147, 196-230) between the caller's 2D-2D matcher and the
 * crop above: each reference view's matches, cv2.estimateAffinePartial2D on the view with the most, the box of its corners.
 * Caller's current device and stream, device pointers, asynchronous, no host synchronisation, no allocation.
 *
 * cv2.estimateAffinePartial2D(from, to, method=RANSAC, threshold, max_iters, confidence, refine_iters) for B independent
 * problems; problem b is pairs offsets[b] .. offsets[b+1] - 1.
 *   from, to      device fp32 [sum n, 2]   the point pairs (cv2 converts its input to fp32 too)
 *   offsets       device int32 [B + 1]
 *   threshold     ransacReprojThreshold (finite); max_iters >= 0; 0 < confidence < 1; refine_iters >= 0
 *   affine        device f64 [B, 6] out    row-major 2x3 [a -b tx; b a ty]; zeros where cv2 returns None
 *   inlier_mask   device uint8 [sum n] out, or NULL: cv2's inlier mask (all zeros where it returns None)
 *   iterations    device int32 [B] out     iterations of the RANSAC loop (0 for n <= 2)
 *   status        device int32 [B] out     1: a model, 0: none (cv2's None)
 * OpenCV's algorithm stage for stage (OpenCV 4.13; the model is tests/affine_ransac_reference.py): n < 2 has no model, n == 2
 * is the one 2-pair model with both pairs inliers (it may be non-finite, as cv2's is); otherwise the samples of
 * cv::RNG((uint64)-1) by getSubset (2 distinct indices), each one's closed-form similarity in fp64 from the fp32 points, the
 * fp32 error ((F0 x + F1 y) + F2 - X)^2 + (...)^2 with the model rounded to fp32, against (float)(threshold^2), every operation
 * rounded on its own; a sample wins when its count exceeds max(best, 1), and each win lowers the budget to
 * RANSACUpdateNumIters(confidence, outlier ratio, 2, budget).  The winner's inliers are refined by OpenCV's LMSolver on
 * (a, b, tx, ty) for at most refine_iters iterations, kept steps or not: its damping schedule (lambda from 1, halved to 0 on
 * good steps, raised by nu on poor ones), its stop once every residual of the kept model is below FLT_EPSILON, and its
 * eigen-decomposition solve that drops eigenvalues below 2 DBL_EPSILON * trace (fp64, reductions in a fixed order).  The
 * samples, counts, mask and the unrefined model are cv2's bit for bit; the refined
 * model was measured within 1.7e-13 relative of cv2 4.13's at every refine_iters from 1 to 1000, with coordinates up to 1e6
 * and thresholds up to 1e200 (DESIGN 5.8).  Results do not depend on the launch. */
int opb_estimate_affine_partial(const float* from, const float* to, const int32_t* offsets, int32_t B, double threshold, int32_t max_iters,
                                double confidence, int32_t refine_iters, double* affine, uint8_t* inlier_mask, int32_t* iterations,
                                int32_t* status, void* stream);
/* match_worker + detect_by_matching (local_feature_2D_detector.py:76-147) for B frames against V reference views.
 *   ref_keypoints    device fp32 [V, cap_ref, 2]  the views' key points (x, y); cap_ref <= 8192
 *   ref_counts       device int32 [V]             key points of view v (entries past it are ignored)
 *   ref_sizes        device int32 [V, 2]          the view's image (H, W)
 *   query_keypoints  device fp32 [B, cap_query, 2], query_counts device int32 [B]
 *   matches0         device int32 or int64 (matches_int64 = 1) [B, V, cap_ref]: the matcher's matches0 of frame b against
 *                    view v; entry i is a match iff 0 <= m < query_counts[b]
 *   query_h, query_w the frames' size.  1 <= V <= 256.
 *   box              device int32 [B, 4] out     [x0, y0, x1, y1], the input of opb_crop_resize
 *   view             device int32 [B] out        the chosen view;  n_matches  device int32 [B] out  its match count
 *   affine           device f64 [B, 6] out       its cv2.estimateAffinePartial2D(ref, query, ransacReprojThreshold=6) model
 *   status           device int32 [B] out        1: the box of the affine; 2: no view has 6 matches, the box is
 *                                                [0, 0, query_h, query_w]; 0: the empty box (see below)
 * Per frame: the views with at least 6 matches compete on their match count, the first view wins a tie (Python's stable sort
 * on inliers.shape[0], which is the match count); no such view: the first view's [0, 0, size[0], size[1]] box, i.e. x1 = H and
 * y1 = W as the reference writes it.  The winner's pairs, in ascending reference key-point order, go through the estimator
 * above with the reference's arguments (threshold 6, 2000 iterations, confidence 0.99, 10 refinement steps); its model maps
 * the view's corners (0, 0), (W, 0), (0, H), (W, H) in fp64 (products summed in index order), truncated to int32, then min /
 * max.  The empty box [0, 0, 0, 0], which opb_crop_resize rejects, where the reference fails: the estimator finds no model
 * (the reference raises a TypeError), or a corner is non-finite or outside int32 (numpy's cast is undefined).  The trace of
 * opb_debug_set_affine_trace records the winning view's loop. */
int opb_boxes_from_matches(const float* ref_keypoints, const int32_t* ref_counts, const int32_t* ref_sizes, int32_t V, int32_t cap_ref,
                           const float* query_keypoints, const int32_t* query_counts, int32_t cap_query, const void* matches0,
                           int32_t matches_int64, int32_t B, int32_t query_h, int32_t query_w, int32_t* box, int32_t* view,
                           int32_t* n_matches, double* affine, int32_t* status, void* stream);
/* opb_boxes_from_matches for B (frame, object) pairs in one launch, each object against its own reference views.
 *   ref_keypoints, ref_counts, ref_sizes   the views of every object in one table: [n_views, cap_ref, 2], [n_views], [n_views, 2]
 *   view_first, view_count   device int32 [B]: pair b's object is views view_first[b] .. view_first[b] + view_count[b] - 1
 *   V_max                    the matches0 row stride, 1 <= V_max <= 256; view_count[b] <= V_max
 *   query_keypoints          device fp32 [n_query, cap_query, 2], query_counts device int32 [n_query]: one row per frame
 *   query_index              device int32 [B]: the query row of pair b, so a frame shared by several pairs is extracted once
 *   matches0                 device int32 or int64 [B, V_max, cap_ref]: row [b, v] is the matcher's matches0 of pair b's frame
 *                            against its object's view v (entries past view_count[b] are never read)
 *   query_h, query_w, box, view, n_matches, affine, status   as in opb_boxes_from_matches; view is the index among pair b's
 *                            object's views.
 * Pair b's results equal, bit for bit, those of opb_boxes_from_matches on its object's views alone and its frame's row, and
 * the trace of opb_debug_set_affine_trace records them as problem b.  A pair whose view range leaves [0, n_views) or whose
 * view_count is outside [1, V_max] or whose query_index is outside [0, n_query) gets status 0, the empty box, view 0,
 * n_matches 0 and a zero affine. */
int opb_boxes_from_matches_objects(const float* ref_keypoints, const int32_t* ref_counts, const int32_t* ref_sizes, int32_t n_views,
                                   int32_t cap_ref, const int32_t* view_first, const int32_t* view_count, int32_t V_max,
                                   const float* query_keypoints, const int32_t* query_counts, int32_t n_query, int32_t cap_query,
                                   const int32_t* query_index, const void* matches0, int32_t matches_int64, int32_t B, int32_t query_h,
                                   int32_t query_w, int32_t* box, int32_t* view, int32_t* n_matches, double* affine, int32_t* status,
                                   void* stream);
/* Test hook of the three calls above: device buffers later calls fill (NULL to stop), per problem b and for every sample i <
 * capacity the loop evaluates: samples int32 [B][capacity][2], counts int32 [B][capacity], models f64 [B][capacity][6] (the
 * unrefined 2-pair model, row-major 2x3). */
int opb_debug_set_affine_trace(int32_t* samples, int32_t* counts, double* models, int32_t capacity);

/* ---- the tracker's flow step: an object's keyframe points followed into the next crop (ba_tracker.py:113-126, 295-356) ----
 * Caller's current device and stream, device pointers, asynchronous, no host synchronisation, no allocation.
 *
 * cv2.calcOpticalFlowPyrLK(prev[b], next[b], pts, None, winSize=(win_w, win_h), maxLevel=max_level,
 * criteria=(criteria_type, max_count, epsilon), flags=0, minEigThreshold=min_eig_threshold) for B image pairs:
 *   prev, next    device uint8 [B, H, W] grey images with the given frame and row pitches in bytes (row pitch >= W)
 *   sizes         device int32 [B, 2] = (h_b, w_b) <= (H, W): pair b's images are the top-left h_b x w_b of its slots (an entry
 *                 outside [1, H] x [1, W] is clamped into it); NULL: every pair is H x W.  H, W <= 32767, B <= 65535
 *   pts, offsets  device fp32 [total, 2] (x, y), int32 [B + 1]: pair b owns rows offsets[b] .. offsets[b + 1] - 1, offsets[0] =
 *                 0 and offsets[B] = total
 *   win_w, win_h  odd, 3 .. 31;  max_level 0 .. 4 (fewer levels where cv2 builds fewer: see the pyramid below)
 *   criteria_type 1 (COUNT), 2 (EPS) or 3; max_count 1 .. 100 with COUNT (30 without), epsilon >= 0 with EPS (0.01 without;
 *                 clamped to 10); flags must be 0 (OPTFLOW_USE_INITIAL_FLOW and OPTFLOW_LK_GET_MIN_EIGENVALS are refused)
 *   workspace     device, 16-byte aligned, at least opb_optical_flow_workspace_bytes(B, H, W, max_level) bytes (a misaligned
 *                 workspace is refused); after the call it holds the
 *                 pyramids: per pair a slot of pair_bytes = that size / B, and in it per level l = 0 .. max_level of an
 *                 H x W pyramid (h_l = ceil(h_{l-1} / 2), likewise w_l) the Scharr derivatives of prev int16 [h_l, w_l, 2],
 *                 then for l >= 1 prev and next uint8 [h_l, w_l], each starting at a multiple of 16 bytes.  A smaller pair
 *                 fills the top-left corner of each level (row pitch w_l); levels past its last are not written.
 *   next_pts, status, err   device fp32 [total, 2], uint8 [total], fp32 [total] out
 * The results are cv2's, bit for bit for status, points and err (OpenCV 4.13; the model is tests/lk_reference.py):
 *   pyramid      level l+1 = cv2.pyrDown(level l), BORDER_REFLECT_101; a pair stops after level l when level l+1 would have a
 *                side <= the window's (cv2.buildOpticalFlowPyramid's return value)
 *   derivatives  cv2.Scharr dx / dy of each prev level as int16, BORDER_REFLECT_101; windows read images through
 *                BORDER_REFLECT_101 and derivatives through a zero border
 *   per point    from the coarsest level: 14-bit bilinear weights, the structure tensor and mismatch vector summed in fp32 in
 *                OpenCV's SIMD order, the minimum-eigenvalue test, up to max_count Newton steps (stop at |d|^2 <= eps^2, or
 *                half a step back when two steps cancel to < 0.01), the guess doubled level to level
 *   status       0 for a point that starts or ends outside the level-0 image or fails the eigenvalue test at level 0
 *   err          mean |next - prev| over the window in grey levels; 0 where status is 0 (cv2 leaves it unset there) */
int opb_optical_flow_workspace_bytes(int32_t B, int32_t H, int32_t W, int32_t max_level, int64_t* bytes);
int opb_calc_optical_flow_pyr_lk(const uint8_t* prev, int64_t prev_frame_pitch, int64_t prev_row_pitch, const uint8_t* next,
                                 int64_t next_frame_pitch, int64_t next_row_pitch, int32_t B, int32_t H, int32_t W, const int32_t* sizes,
                                 const float* pts, const int32_t* offsets, int32_t total, int32_t win_w, int32_t win_h, int32_t max_level,
                                 int32_t criteria_type, int32_t max_count, double epsilon, double min_eig_threshold, int32_t flags,
                                 void* workspace, int64_t workspace_bytes, float* next_pts, uint8_t* status, float* err, void* stream);
/* np.where(status == 1) of B tracks, kpt_flow_track's valid ids (ba_tracker.py:122-124) applied to both point lists:
 *   status, pts2d, pts3d   device uint8 [B, cap], fp32 [B, cap, 2], fp32 [B, cap, 3]; track b's rows are 0 .. counts[b] - 1
 *   counts                 device int32 [B] (clamped to [0, cap])
 *   out2d, out3d           device f64 [B * cap, 2], [B * cap, 3] out: the kept rows, track-major, in row order
 *   offsets, n_tracked     device int32 [B + 1], [B] out: track b's kept rows are offsets[b] .. offsets[b + 1] - 1
 *   pad2d, pad3d           device fp32 [B, cap, 2], [B, cap, 3] out: track b's kept rows first, then zeros */
int opb_flow_compact(const uint8_t* status, const float* pts2d, const float* pts3d, const int32_t* counts, int32_t B, int32_t cap,
                     double* out2d, double* out3d, int32_t* offsets, int32_t* n_tracked, float* pad2d, float* pad3d, void* stream);
/* flow_track's kpt_dist (ba_tracker.py:326-327): per track b, the fp64 mean over rows offsets[b] .. offsets[b + 1] - 1 of
 * |project(pts3d, K[b], pose[b]) - pts2d| (tracking_utils.project: X R^T + t, then K, then x / z); NaN for a track without
 * rows.  K f64 [B, 9], pose f64 [B, 12] (row-major 3x4), pts2d f64 [n, 2], pts3d f64 [n, 3], dist f64 [B] out. */
int opb_flow_reprojection(const double* K, const double* pose, const double* pts2d, const double* pts3d, const int32_t* offsets, int32_t B,
                          double* dist, void* stream);

/* ---- an object's SfM post-processing (csrc/sfm.cu) ----
 * run.py postprocess (:142-163) after COLMAP's triangulation: get_tkl and filter_3d, merge, and the 3D half of get_kpt_ann.
 * Caller's current device and stream, device pointers, asynchronous, no host synchronisation, no allocation: each step sizes
 * one caller-provided workspace (256-byte aligned) with its *_workspace_bytes query.  A count one step finds (kept points,
 * groups, observations) is written to a device int64 that the next step reads; `cap` arguments bound what a step may hold.
 *
 * opb_sfm_filter_points: P points in ascending id order, ids int64 [P], xyz f64 [P, 3], track_len int64 [P] (COLMAP's
 * point2D_idxs lengths); corners f64 [8, 3]; max_num_kp3d >= 0.
 *   track_length  out: get_tkl's threshold, the smallest length L present with at most max_num_kp3d points longer than L (the
 *                 group at L is kept whole, so more than max_num_kp3d points can pass)
 *   kept_ids, kept_xyz   int64 [P], fp32 [P, 3] out: the points of length >= track_length strictly inside the box, in order;
 *                 filter_by_3d_box in fp32: m = (p - c4) . v for v = c5 - c4, c0 - c4, c7 - c4, kept when 0 < m < v . v,
 *                 each product and sum rounded on its own, the sums left to right
 *   n_kept        out: the kept count */
int opb_sfm_filter_workspace_bytes(int32_t P, int64_t* bytes);
int opb_sfm_filter_points(const int64_t* ids, const double* xyz, const int64_t* track_len, int32_t P, int32_t max_num_kp3d,
                          const double* corners, void* workspace, int64_t workspace_bytes, int64_t* kept_ids, float* kept_xyz,
                          int64_t* track_length, int64_t* n_kept, void* stream);
/* opb_sfm_merge_points: merge (filter_points.py:86-117) of the first min(*n, cap) rows of xyz fp32 [cap, 3] with ids int64.
 * Point i neighbours j when scipy's pdist of their rows widened to fp64 (dx*dx + dy*dy, + dz*dz, correctly rounded sqrt) is
 * below dist_threshold (> 0); j neighbours itself.  The greedy pass walks j in order: j is skipped when any neighbour is already
 * in a group, otherwise its neighbours, ascending, are the next group.  A point can be dropped without being in any group.
 *   merged_xyz     f64 [cap, 3] out   np.mean of the group's fp32 rows (fp32 sum in member order, fp32 divide), widened
 *   group_offsets  int32 [cap + 1] out  group g's members are group_offsets[g] .. group_offsets[g + 1] - 1
 *   member_ids, member_index   int64 / int32 [cap] out: each member's id and row
 *   slot_of        int32 [cap] out    row i's member position, or INT32_MAX for a row in no group
 *   n_groups, n_members   out: the groups and their members (group_offsets[n_groups]); nothing is written past row
 *                  min(*n, cap) - 1 of member_ids, member_index or slot_of */
int opb_sfm_merge_workspace_bytes(int32_t cap, int64_t* bytes);
int opb_sfm_merge_points(const float* xyz, const int64_t* ids, const int64_t* n, int32_t cap, double dist_threshold, void* workspace,
                         int64_t workspace_bytes, double* merged_xyz, int32_t* group_offsets, int64_t* member_ids, int32_t* member_index,
                         int32_t* slot_of, int64_t* n_groups, int64_t* n_members, void* stream);
/* opb_sfm_gather_observations: the observations of the merge groups in get_kpt_ann's order.  Image f (the caller's order) holds
 * features 0 .. counts[f] - 1 (counts[f] <= cap) whose COLMAP point ids are point3d_ids int64 [F, cap] (-1: none); F * cap
 * <= INT32_MAX.  A feature observes member m when its id is kept_ids[i] (ascending, the first min(*n_kept, kept_cap)) and
 * slot_of[i] = m (opb_sfm_merge_points' outputs).
 *   order    int32 [F * cap] out   the observing features as f * cap + k, ordered by member position and, within a member,
 *                                  by (image, feature); one image may observe a point twice
 *   idxs     int64 [kept_cap] out  each group's observation count
 *   total    out: the number of observations (the valid prefix of order)
 *   missing  out: the position of the first member without an observation (the reference's KeyError), or a value above
 *            every position */
int opb_sfm_gather_workspace_bytes(int32_t F, int32_t cap, int32_t kept_cap, int64_t* bytes);
int opb_sfm_gather_observations(const int64_t* point3d_ids, const int32_t* counts, int32_t F, int32_t cap, const int64_t* kept_ids,
                                const int64_t* n_kept, int32_t kept_cap, const int32_t* slot_of, const int32_t* group_offsets,
                                const int64_t* n_groups, void* workspace, int64_t workspace_bytes, int32_t* order, int64_t* idxs,
                                int64_t* total, int64_t* missing, void* stream);
/* opb_sfm_gather_features: rows 0 .. total - 1 of the collected features, widened to f64: out_descriptors [total, D] row r =
 * descriptors[f, :, k] and out_scores [total] = scores[f, k] for order[r] = f * cap + k.  scores fp32 [F, cap], descriptors
 * fp32 [F, D, cap] (SuperPoint's padded outputs). */
int opb_sfm_gather_features(const int32_t* order, int64_t total, int32_t F, int32_t cap, int32_t D, const float* scores,
                            const float* descriptors, double* out_descriptors, double* out_scores, void* stream);
/* opb_sfm_assign_pairs: each image's assign matrix (count_features and get_assign_matrix, feature_process.py:95-135,
 * :197-230).  Image f holds features 0 .. counts[f] - 1 with COLMAP point ids point3d_ids int64 [F, cap] (-1: none), cap <=
 * OPB_SFM_ASSIGN_MAX_CAP (one image is one block's shared memory).  A feature's id is kept when it is in kept_ids int64 [M]
 * (ascending, distinct) and then belongs to group kept_group[i] (0 <= group < M).  Per image, in the order of each group's first
 * feature k0: (the last feature whose id is k0's, the group) -- one pair per group.
 *   pairs        int64 [2, F * cap] out   row 0 the features, row 1 the groups; image f's pairs are columns offsets[f] ..
 *                                         offsets[f + 1] - 1 (columns past offsets[F] are not written)
 *   offsets      int64 [F + 1] out
 *   num_matches  int64 [F] out */
#define OPB_SFM_ASSIGN_MAX_CAP 8192
int opb_sfm_assign_workspace_bytes(int32_t F, int32_t cap, int64_t* bytes);
int opb_sfm_assign_pairs(const int64_t* point3d_ids, const int32_t* counts, int32_t F, int32_t cap, const int64_t* kept_ids,
                         const int32_t* kept_group, int32_t M, void* workspace, int64_t workspace_bytes, int64_t* pairs, int64_t* offsets,
                         int64_t* num_matches, void* stream);

/* ---- the JSON text of the per-image 2D annotation files (csrc/json_text.cu) ----
 * save_2d_anno_for_each_image's json.dump (feature_process.py:233-262): {"keypoints2d": [n, 2], "descriptors2d": [D, n],
 * "scores2d": [n, 1], "assign_matrix": [2, k], "num_matches": k} with ", " and ": ", each fp32 feature as float.__repr__ of the
 * widened double (NaN, Infinity, -Infinity as json writes them) and the integers as int.__repr__.
 *
 * opb_json_float_repr: float.__repr__ of (double)x[i] into out [n, 24] (NUL-padded) and its length into len int32 [n].
 * opb_json_float_repr_host: the same routine on the host, on host memory.
 *
 * A chunk of Fc <= 65535 images: images int64 [Fc, 4] = (feature row f, n, k >= 1, pair offset) per image, device memory; image c's
 * numbers are keypoints fp32 [F, cap, 2] row f, descriptors fp32 [F, D, cap] row f, scores fp32 [F, cap] row f, both rows of
 * pairs int64 [2, pair_stride] from the pair offset (opb_sfm_assign_pairs' layout) and k.  Its text is 3n + Dn + 2k + 1 items
 * (a number and the text before it; the last one closes the object); item_off int64 [Fc + 1] gives the chunk's first item of
 * each image, items = item_off[Fc], and max_items >= every image's item count, at most OPB_ANNO2D_MAX_IMAGE_ITEMS.
 * opb_anno2d_text_lengths sizes every item into the workspace and writes offsets int64 [Fc + 1] (device): image c's text is
 * bytes offsets[c] .. offsets[c + 1] - 1 of the chunk's.  opb_anno2d_text_write then writes the text to out (offsets[Fc] bytes)
 * from the same arguments, the workspace that opb_anno2d_text_lengths filled and its offsets. */
#define OPB_ANNO2D_MAX_IMAGE_ITEMS (1 << 24)
int opb_json_float_repr(const float* x, int64_t n, char* out, int32_t* len, void* stream);
int opb_json_float_repr_host(const float* x, int64_t n, char* out, int32_t* len);
int opb_anno2d_text_workspace_bytes(int32_t Fc, int64_t items, int64_t* bytes);
int opb_anno2d_text_lengths(const int64_t* images, const int64_t* item_off, int32_t Fc, int64_t items, int64_t max_items, int32_t D,
                            int32_t cap, const float* keypoints, const float* descriptors, const float* scores, const int64_t* pairs,
                            int64_t pair_stride, void* workspace, int64_t workspace_bytes, int64_t* offsets, void* stream);
int opb_anno2d_text_write(const int64_t* images, const int64_t* item_off, int32_t Fc, int64_t max_items, int32_t D, int32_t cap,
                          const float* keypoints, const float* descriptors, const float* scores, const int64_t* pairs, int64_t pair_stride,
                          const void* workspace, const int64_t* offsets, char* out, void* stream);

/* ---- PNG files of camera frames and crops (csrc/png.cu) ----
 * The bytes cv2.imencode('.png', frame) (OpenCV 4.13's default call) writes for 8-bit frames, as parse_scanned_data.py's
 * cv2.imwrite of color/ and color_full/ does (:173, :177, :264-273): SUB-filtered rows (NONE when W = 1), zlib 1.3's level 1
 * Z_RLE deflate at memLevel 8 with libpng's window and header, IDAT chunks of 8192 bytes with their CRC-32, no ancillary
 * chunks.  The model is tests/png_reference.py and DESIGN §5.15 states the rules.
 *
 * opb_png_encode: F frames of one shape in one call, on the caller's stream, with no allocation and no host synchronisation.
 *   frames     device uint8 [F, H, W, C], C = 1 (grey), 3 (BGR) or 4 (BGRA) in cv2's channel order; frame f starts at frames +
 *              f * frame_pitch, its row y at + y * row_pitch (bytes; row_pitch >= W * C; frame_pitch 0, one frame for all F, or
 *              >= H * row_pitch).  F <= OPB_PNG_MAX_FRAMES, H * (1 + W * C) <= 2^28.
 *   workspace  device, 256-byte aligned, at least opb_png_workspace_bytes(F, H, W, C); its contents on entry do not matter
 *   out        device uint8 [F, out_pitch]: frame f's file at out + f * out_pitch, out_pitch >= opb_png_frame_bytes(H, W, C)
 *              (zlib's deflateBound of the H * (1 + W * C) filtered bytes, 12 bytes per IDAT chunk and 45 for the signature,
 *              IHDR and IEND); bytes past a file's size are not written
 *   sizes      device int64 [F] out: each file's size in bytes, or -1 for a file that would not fit its slot (nothing of it is
 *              then written) */
#define OPB_PNG_MAX_FRAMES 65535
int opb_png_workspace_bytes(int32_t F, int32_t H, int32_t W, int32_t C, int64_t* bytes);
int opb_png_frame_bytes(int32_t H, int32_t W, int32_t C, int64_t* bytes);
int opb_png_encode(const uint8_t* frames, int64_t frame_pitch, int64_t row_pitch, int32_t F, int32_t H, int32_t W, int32_t C,
                   void* workspace, int64_t workspace_bytes, uint8_t* out, int64_t out_pitch, int64_t* sizes, void* stream);

/* ---- PNG files read as cv2.imread / cv2.imdecode read them (csrc/png_decode.cu) ----
 * Every stage of the reference reads its frames and crops with cv2.imread: NormalizedDataset (src/datasets/
 * normalized_dataset.py:25-34) and the SfM feature extraction with IMREAD_GRAYSCALE, the detector's views and queries
 * (local_feature_2D_detector.py:155, :173), data_utils.read_gray_scale.  opb_png_decode gives OpenCV 4.13's pixels (libpng 1.6,
 * zlib 1.3) for 8-bit grey (colour type 0), RGB (2) and RGBA (6) files that are not interlaced: any zlib stream (stored, fixed
 * and dynamic blocks, any window) in any split into IDAT chunks, every row filter.  DESIGN §5.16 states the rules and the model
 * is tests/png_decode_reference.py.
 *
 * F files of one width and height in one call, on the caller's stream, with no allocation and no host synchronisation.
 *   data       device bytes of the files back to back; file f is data[offsets[f] .. offsets[f + 1])
 *   offsets    device int64 [F + 1], non-decreasing from 0, offsets[F] <= the total_bytes the workspace was sized for (a file
 *              outside it reports OPB_PNG_NOT_PNG; offsets that decrease anywhere make every file report OPB_PNG_NOT_PNG)
 *   F, H, W    F <= OPB_PNG_MAX_FRAMES, H * (1 + 4 W) <= 2^28; every file's IHDR must give W x H
 *   mode       OPB_PNG_READ_GREY: IMREAD_GRAYSCALE, uint8 [H, W] pixels (a grey file's own, else
 *              (9797 R + 19234 G + 3737 B) >> 15 with alpha ignored, as opb_grey_frames);
 *              OPB_PNG_READ_BGR: IMREAD_COLOR, uint8 [H, W, 3] BGR (grey replicated, alpha dropped)
 *   workspace  device, 256-byte aligned, at least opb_png_decode_workspace_bytes(F, H, W, total_bytes); contents on entry do
 *              not matter
 *   out        device: file f's pixel (y, x) at out + f * out_frame_pitch + y * out_row_pitch + x * (1 or 3) (out_row_pitch >=
 *              W * (1 or 3), out_frame_pitch >= H * out_row_pitch when F > 1)
 *   image      NULL, or with OPB_PNG_READ_GREY device fp32 [F, 1, H, W] (dense): grey / 255 as a float32 division
 *   status     device int32 [F] out: OPB_PNG_* below.  A file whose status is not OPB_PNG_OK has none of its out / image
 *              pixels written; cv2.imdecode returns None for every such file, and an image for every OPB_PNG_OK file.
 * Statuses: OPB_PNG_NOT_PNG (signature, chunk structure, order or an unhandled critical chunk), OPB_PNG_BAD_CRC (a critical
 * chunk's CRC-32; an ancillary chunk's is only a warning), OPB_PNG_UNSUPPORTED (another bit depth, colour type, interlace, or
 * a colour file read grey with gAMA != 1.0, sRGB or iCCP, where libpng converts in linear light), OPB_PNG_BAD_SHAPE (IHDR is not
 * W x H), OPB_PNG_BAD_DEFLATE (what zlib rejects), OPB_PNG_BAD_ADLER, OPB_PNG_TOO_LITTLE_DATA (the stream ends before the
 * last row), OPB_PNG_BAD_FILTER (a row filter byte > 4). */
enum { OPB_PNG_READ_GREY = 0, OPB_PNG_READ_BGR = 1 };
enum {
  OPB_PNG_OK = 0, OPB_PNG_NOT_PNG = 1, OPB_PNG_BAD_CRC = 2, OPB_PNG_UNSUPPORTED = 3, OPB_PNG_BAD_SHAPE = 4, OPB_PNG_BAD_DEFLATE = 5,
  OPB_PNG_BAD_ADLER = 6, OPB_PNG_TOO_LITTLE_DATA = 7, OPB_PNG_BAD_FILTER = 8
};
int opb_png_decode_workspace_bytes(int32_t F, int32_t H, int32_t W, int64_t total_bytes, int64_t* bytes);
int opb_png_decode(const uint8_t* data, const int64_t* offsets, int32_t F, int32_t H, int32_t W, int32_t mode, void* workspace,
                   int64_t workspace_bytes, uint8_t* out, int64_t out_frame_pitch, int64_t out_row_pitch, float* image,
                   int32_t* status, void* stream);

/* ---- the tracker's flow-only state machine (csrc/track.cu) ----
 * BATracker's per-frame logic around flow_track in the live demo's order (inference_demo.py:253-299, track_interval 5) with
 * track(frame, flow_track_only=True): update_kf's gate, add_kf's first pose, motion_prediction and track()'s choice of the
 * pose (src/tracker/ba_tracker.py:105-145, :147-149, :275-293, :727-802).  One thread per track in fp64, on the caller's
 * stream, no allocation and no host synchronisation.  Bundle adjustment is not part of it.
 *
 * Per-track state, device memory the caller owns (onepose_b200.track.init_state makes it):
 *   frame            int64 [B]        frames seen (the demo's id); 0 for a new or reset track
 *   hist             f64 [B, 3, 16]   the last up to 3 reported poses (pose_list[-3:]), row-major 4x4, oldest first
 *   hist_len         int32 [B]        poses in hist, 0..3
 *   init_cnt         int32 [B]        init_cnt, 3 for a new track
 *   use_motion_cnt   int32 [B]        use_motion_cnt, 0 for a new track
 * A track is at its first frame when frame <= 0 or hist_len <= 0.  Poses are row-major 4x4 f64 [B, 16]. */
enum { OPB_TRACK_GATE_NONE = 0, OPB_TRACK_GATE_ADD = 1, OPB_TRACK_GATE_ACCEPT = 2, OPB_TRACK_GATE_REJECT = 3 };
enum { OPB_TRACK_FLOW = 0, OPB_TRACK_MOTION = 1, OPB_TRACK_PRED = 2, OPB_TRACK_INIT = 3, OPB_TRACK_KEYFRAME = 4 };
/* The keyframe decision of this frame, per track: GATE_ADD at the first frame (update_kf accepts with no keyframe, then add_kf;
 * hist becomes [pose_pred], hist_len 1); at frame % 5 == 0 GATE_REJECT if cm_degree_5_metric(pose_pred, last reported pose)
 * has trans > 10 cm or rot > 10 deg, else GATE_ACCEPT (the frame's inlier pairs become the keyframe); GATE_NONE otherwise.
 * pose_pred f64 [B, 16] (the frame's matcher pose), gate int32 [B] out.  Only the first frame writes hist / hist_len. */
int opb_track_gate(const double* pose_pred, int32_t B, const int64_t* frame, double* hist, int32_t* hist_len, int32_t* gate, void* stream);
/* track()'s steps 2-6 after flow_track, per track: with d = cm_degree_5_metric(last reported pose, pose_flow) and pose_mo =
 * pose_pred while hist_len < 3, else motion_prediction(hist): pose_mo if ((d.trans > 10 or d.rot > 10) and use_motion_cnt < 3)
 * or kpt_dist > 10 (use_motion_cnt + 1); else pose_flow if d.trans < 20 and d.rot < 20 (use_motion_cnt = 0); else pose_mo
 * (use_motion_cnt + 1).  Then while init_cnt > 0 it is decremented and pose_pred reported instead.  The reported pose is
 * appended to hist; a comparison with NaN is false.  At the first frame (no track() call in the demo) pose_out = pose_pred,
 * branch KEYFRAME and only frame changes.  frame += 1 for every track.
 * pose_pred, pose_flow f64 [B, 16] (flow_track's pose_init_homo), kpt_dist f64 [B]; pose_out f64 [B, 16] and branch int32 [B]
 * out (FLOW, MOTION, PRED: pose_mo while the history is short, INIT: the init override, KEYFRAME). */
int opb_track_select(const double* pose_pred, const double* pose_flow, const double* kpt_dist, int32_t B, int64_t* frame, double* hist,
                     int32_t* hist_len, int32_t* init_cnt, int32_t* use_motion_cnt, double* pose_out, int32_t* branch, void* stream);

/* ---- adjacent producer: SuperPoint key-point extractor (SURVEY 8f N4) ----
 * Replaces SuperPoint.forward (reference src/models/extractors/SuperPoint/superpoint.py:140-197): shared VGG-style encoder
 * (:142-152), score head + 65-way softmax + 8x8 pixel shuffle (:155-160), simple_nms (:47-61, :161), threshold / border /
 * top-k key-point selection (:163-174), descriptor head (:180-181) and bilinear descriptor sampling (:79-92, :184-185).
 * Its outputs are the `keypoints2d` / `descriptors2d_query` tensors inference.py:80-94 packs for the matcher; with a fixed
 * capacity (max_keypoints >= 0) they stay on the device: descriptors [B, 256, cap] + counts [B] are exactly the
 * `desc2d_query` / `n2d_lengths` arguments of opb_forward. */
typedef struct opb_superpoint opb_superpoint; /* opaque */

/* = the `config` mapping of SuperPoint.__init__ merged over its default_config (superpoint.py:97-103).  Note that the released
 * inference configuration (src/sfm/extract_features.py:19-24) spells the threshold key 'keypoints_threshold', so the default
 * 0.005 is what the reference runs with; nms_radius 3, max_keypoints 4096. */
typedef struct opb_sp_config {
  int32_t descriptor_dim;     /* 256 (only value supported)                                                    */
  int32_t nms_radius;         /* 0..6                                                                          */
  float keypoint_threshold;   /* superpoint.py:164                                                             */
  int32_t max_keypoints;      /* > 0, or -1 = keep all (superpoint.py:133-135 raises for 0 and < -1)            */
  int32_t remove_borders;     /* superpoint.py:64-69                                                           */
  int32_t align_corners;      /* grid_sample flag: 1 under the reference's pinned torch 1.8 (superpoint.py:86)  */
  int32_t device;
} opb_sp_config;

int opb_sp_create(const opb_sp_config* cfg, opb_superpoint** out);
void opb_sp_destroy(opb_superpoint* h);
const char* opb_sp_last_error(const opb_superpoint* h); /* h may be NULL: as opb_last_error(NULL) */
/* Reference state-dict keys ("conv1a.weight", "conv1a.bias", ... "convDb.bias"; superpoint.py:111-126), HOST fp32 arrays in
 * the reference's own [C_out, C_in, kh, kw] layout.  opb_sp_finalize_weights packs them (tap-major reduction index, the two
 * heads' 3x3 layers side by side, fp16 hi/lo split) and uploads. */
int opb_sp_load_weight(opb_superpoint* h, const char* name, const float* data, size_t n_elems);
int opb_sp_finalize_weights(opb_superpoint* h);
/* First half of forward(): image device fp32 [B, 1, H, W] (H, W multiples of 8) -> internal candidate lists.
 * counts (device int32 [B], may be NULL) receives the number of key points opb_sp_describe will emit for each image
 * (= min(#candidates, max_keypoints)); a caller that needs exactly-sized outputs reads it (the reference synchronises at the
 * same point: torch.nonzero, superpoint.py:163-165) and passes cap = max(counts). */
int opb_sp_detect(opb_superpoint* h, const float* image, int32_t B, int32_t H, int32_t W, int32_t* counts, void* stream);
/* Second half: key points (x, y) fp32 [B, cap, 2], scores fp32 [B, cap], descriptors fp32 [B, 256, cap] (channel-first like the
 * reference's [256, n]; may be NULL), counts int32 [B]; entries >= counts[b] are not written.  Order: row-major (torch.nonzero)
 * or, when an image has more than max_keypoints candidates, descending score (torch.topk). */
int opb_sp_describe(opb_superpoint* h, float* keypoints, float* scores, float* descriptors, int32_t* counts, int32_t cap, void* stream);
/* Both halves with a caller-chosen capacity, no host synchronisation (cap >= max_keypoints makes it exact). */
int opb_sp_forward(opb_superpoint* h, const float* image, int32_t B, int32_t H, int32_t W, float* keypoints, float* scores,
                   float* descriptors, int32_t* counts, int32_t cap, void* stream);
/* Range guard of the fp16-split operand format (|x| < 1023 per plane element), as for the matcher.  conv1a and every 3x3
 * convolution check what they split: a value at |x| >= 1023 (after the ReLU), or an inf / NaN image pixel, raises a flag.
 * opb_sp_finalize_weights refuses (OPB_E_RANGE) a weight or bias that is not finite, or a weight of a tensor-core layer
 * (all but conv1a) at |w| >= 1023; with those excluded no NaN can arise that the check would not see.  A call that raised
 * the flag reports count 0 for every image, on the device and without blocking, and the error is delivered to the host
 * lazily:
 *   opb_sp_poll_range   never blocks: OPB_E_RANGE if a finished earlier call raised the flag, OPB_OK otherwise (also while
 *                       the last call is still running).  opb_sp_detect (and so opb_sp_forward) calls it first, and returns
 *                       its error without running;
 *   opb_sp_check_range  waits for the handle's last call and reports.
 * Reporting clears the flag; the clearing is ordered before the handle's next call, on whatever stream. */
int opb_sp_check_range(opb_superpoint* h, void* stream);
int opb_sp_poll_range(opb_superpoint* h);
int opb_sp_last_launch_count(const opb_superpoint* h);
/* bench.py hooks: with profiling on, an event follows every launch of opb_sp_detect / opb_sp_describe; entry i = launch i
 * (name, milliseconds, algorithmic FLOPs of a convolution: 2 * interior pixels * C_out * 9 * C_in). */
int opb_sp_set_profiling(opb_superpoint* h, int32_t enable);
int opb_sp_get_profile(opb_superpoint* h, int32_t index, char* name, size_t name_cap, double* ms, double* flops);
/* test hooks: stop the encoder after step i (0 conv1a, 1 conv1b, 2 pool, 3 conv2a, 4 conv2b, 5 pool, 6 conv3a, 7 conv3b, 8 pool,
 * 9 conv4a, 10 conv4b, 11 [convPa|convDa]; -1 = run everything) and read internal tensors as fp32: which = 0 dense scores
 * [B,H,W], 1 scores after NMS, 2 convPb output rows [B*P, 128], 3 convDb output rows [B*P, 256], 4 the activation of the last
 * step run, rows of the zero-bordered pixel grid [B*P, C]. */
int opb_sp_debug_set_stop(opb_superpoint* h, int32_t layer);
/* 3x3 convolutions on the 64-wide column tiles: 1 (default) = halo boxes (one (128 + 2)-row A box per kernel row and
 * 64-channel block serves the three horizontal taps through row-offset wgmma descriptors: a third of the L2 -> shared-memory
 * traffic), 0 = nine row-shifted boxes per tile.  Same operand bytes and products: bit-identical results with 64 input channels;
 * with more, the halo form visits (kernel row, channel block, dx) instead of (tap, channel block), equal to fp32 rounding.
 * Wider tiles always use the nine boxes (a halo stage of a 128-wide tile leaves no room for a second stage).  A/B switch for
 * tests/ and tools/. */
int opb_debug_set_conv_halo(int32_t mode);
int opb_sp_debug_read(opb_superpoint* h, int32_t which, float* out, size_t capacity_elems, int64_t* n_elems, void* stream);

/* ---- test hooks (used by tests/ and tools/ only; stable but not part of the drop-in surface) ---- */
/* Stop the next opb_forward / opb_forward_objects right after step `step` of GNN layer `layer` of the chunk chosen by
 * opb_debug_set_stop_pass (default: the first); the call returns OPB_OK and its outputs are unspecified.  layer = -1 turns the hook off (default).  Steps of an attention layer (1, 2,
 * 4, 5, 7, 8, 10, 11): 0 k,v projection, 1 state partials, 2 state reduce, 3 q projection, 4 G fold, 5 mlp.0, 6 InstanceNorm
 * statistics, 7 mlp.3 (+ residual).  A GATs layer (0, 3, 6, 9): 0 aggregation, and with with_linear_transform 1 the W GEMM and
 * its finish.  layer = 12, the tail: 0 final_proj + normalize, 1 score sums, 2 their finalize, 3 score conf.  With hoisting
 * on, layer 1 is the compact query-side pass (the sub-batch chosen by opb_debug_set_stop_pass), and layers 16 / 17 are the
 * object prologue's layers 0 and 1 (the first object whose prologue runs in the call).  A host-side check only: the launches
 * are the same with the hook off. */
int opb_debug_set_stop(opb_matcher* m, int32_t layer, int32_t step);
/* The pass later stops of opb_debug_set_stop apply to: chunk `chunk` of the call (chunks of opb_set_chunk_frames frames) and,
 * for layer 1 with hoisting on, sub-batch `piece` of its query-side pass (16 frames each when the queries come from the host
 * through opb_forward_host, else one per chunk).  The object prologue (layers 16 / 17) ignores both.  Default (0, 0).  A stop
 * the call never reaches leaves the call complete, and opb_debug_read then returns OPB_E_STATE. */
int opb_debug_set_stop_pass(opb_matcher* m, int32_t chunk, int32_t piece);
/* The next forward runs the object prologue of every object of the handle again (with hoisting on), as after a weight reload:
 * a stop at layer 16 / 17 then reaches the prologue of the call's first frame's object. */
int opb_debug_invalidate_prologues(opb_matcher* m);
/* Layout of the pass the last forward stopped in: layout[7] = {B, N, M, n_pad, m_pad, R, S}, rows = B * R, S = 2 B segments
 * (frame b's query rows [b R, b R + n_pad), its 3D rows [b R + n_pad, (b + 1) R)).  OPB_E_STATE if the last forward did not
 * stop. */
int opb_debug_stopped_layout(const opb_matcher* m, int32_t* layout);
/* Copy a buffer of the stopped pass to `out` (device): *n_elems = its size; OPB_E_INVALID when it exceeds capacity_elems.
 * fp32 elements except 12 / 13:  0 X planes [rows, 256], (hi + lo) / 64;  1 kvt [rows, 512] = [elu(K) + 1 | V] (one fp16 plane
 * / 64, head-contiguous channels h*64 + d);  2 Kmean [S, 256];  3 bd [S, 256, 256] (block-diagonal KVmean of the source
 * segment, indexed by destination segment);  4 Q' [rows, 256];  5 G [S, 512, 256];  6 hid (mlp.0 output) [rows, 512];
 * 7 InstanceNorm mean [S, 512];  8 its rstd [S, 512];  9 pn (normalized final_proj rows) [rows, 256];  10 inverse row sums
 * [B, n_pad];  11 inverse column sums [B, m_pad];  12 packed row arg-max int64 [B, N];  13 packed column arg-max int64 [B, M]
 * ((conf bits << 32) | ~index);  14 with_linear_transform only: the GATs rows before W [B * m_pad, 256]. */
int opb_debug_read(opb_matcher* m, int32_t which, void* out, size_t capacity_elems, int64_t* n_elems, void* stream);
/* Programmatic dependent launch on (default) / off for every launch of the library (A/B measurements). */
int opb_debug_set_pdl(int32_t enable);
/* byte >= 0: every workspace / object buffer allocated from now on is filled with `byte` (0xFF = NaN patterns) unless the
 * algorithm requires it to start as zero; -1: off.  Proves that no result depends on uninitialised memory. */
int opb_debug_set_ws_fill(int32_t byte);
/* Tensor-core passes of the k,v projection: 2 (default: A_hi.(B_hi + B_lo); its output is rounded to one fp16 plane anyway) or
 * 3 (the full split product), for the precision A/B in tests/ and tools/. */
int opb_debug_set_kv_passes(opb_matcher* m, int32_t passes);
/* One problem of the GEMM core, field for field the library's own problem description (csrc/gemm_common.cuh GemmProblem):
 *   C[batch][rows, n_out] = [A1 | A2] . [B1 | B2]^T (+ bias) -> the epilogue `epi`
 * Operands are fp16-split planes (hi = fp16(64 x), lo = fp16(64 x - hi); opb_debug_split), row-major, each with its own ld in
 * elements.  Unused pointers are NULL, unused counts 0.  The same rules as the library's own launches apply (rows % 256 == 0,
 * K1, K2 % 64 == 0, ...); a problem the core does not accept returns OPB_E_INVALID. */
typedef struct opb_debug_gemm_desc {
  int32_t epi;              /* 0 fp32 C (+bias), 1 fp32 C + InstanceNorm partials, 2 Q' planes, 5 L2-normalised planes,
                               6 score sums, 7 score conf + arg-maxes, 9 k,v projection, 10 planes = acc + bias, 11 convolution */
  int32_t bn;               /* column-tile width: 0 = 256; 128 (epi 0, 11), 64 (epi 11) */
  int32_t rows;             /* per batch */
  int32_t n_out;
  int32_t K1;
  int32_t K2;               /* 0: no second reduction block */
  int32_t batch;            /* 0 = 1 */
  int64_t a_batch_rows;     /* batch z reads A rows from z * a_batch_rows, B rows from z * b_batch_rows */
  int64_t b_batch_rows;
  const void* a1_hi;        /* [rows, K1] */
  const void* a1_lo;
  int32_t a1_ld;
  const void* a2_hi;        /* [rows, K2] */
  const void* a2_lo;
  int32_t a2_ld;
  const void* b1_hi;        /* [n_out, K1] */
  const void* b1_lo;
  int32_t b1_ld;
  const void* b2_hi;        /* [n_out, K2], or [segments * n_out, K2] per segment */
  const void* b2_lo;
  int32_t b2_ld;
  int32_t b2_mode;          /* 0 shared, 1 one B2 per segment of the layout, 2 the identity with a zero lo plane
                               (converter problems only) */
  int32_t a_hi_only;        /* A enters with its hi plane only (epi 9) */
  const float* a_raw;       /* converter: A1 = ReLU((a_raw - mu[seg]) * rstd[seg]) formed in the core from fp32 [rows, a_raw_ld]; NULL: off */
  int32_t a_raw_ld;
  const float* mu;          /* [segments][512] */
  const float* rstd;
  int32_t B;                /* activation layout: B frames of n_pad query rows + m_pad 3D rows (B = 0: a plain matrix) */
  int32_t N;
  int32_t M;
  int32_t n_pad;
  int32_t m_pad;
  const int32_t* nlen;      /* device [B] valid query rows per frame, or NULL: N */
  const int32_t* mlen;      /* device [B] valid 3D rows per frame, or NULL: M */
  const float* bias;        /* [n_out] or NULL */
  float* c;                 /* epi 0, 1: fp32 [batch * rows, ldc] */
  int32_t ldc;
  void* out_hi;             /* planes out [batch * rows, out_ld] (epi 9: out_hi only, 512 columns) */
  void* out_lo;
  int32_t out_ld;
  const float* kmean;       /* epi 2: [segments][256] */
  int32_t cross;            /* epi 2: source = the other segment of the frame */
  float* statpart;          /* epi 1: [rows / 32][n_out][2] */
  float inv_scale;          /* epi 6, 7 */
  float* rowsum_part;       /* epi 6: [B][2 * n_out / 256][n_pad] */
  float* colsum_part;       /* epi 6: [B][rows / 32][m_pad] */
  const float* inv_rowsum;  /* epi 7: [B][n_pad] */
  const float* inv_colsum;  /* epi 7: [B][m_pad] */
  float* conf;              /* epi 7: [B][N][conf_ld] or NULL */
  int32_t conf_ld;          /* 0 = M */
  uint64_t* rowbest;        /* epi 7: [B][N] packed (conf bits << 32) | ~column */
  uint64_t* colbest;        /* epi 7: [B][M] */
  int32_t taps;             /* epi 11: 1 or 9 row-shifted taps of A (0: plain GEMM) */
  int32_t kb_per_tap;       /* C_in / 64 */
  int32_t tap_off[9];       /* row shift of each tap */
  int32_t cv_w2;            /* epi 11 pixel grid: row r is pixel q = r % cv_ppad, y = q / cv_w2, x = q % cv_w2 */
  int32_t cv_h;
  int32_t cv_w;
  int32_t cv_ppad;
  int32_t relu;
  int32_t* range_flag;      /* epi 11: set to 1 when an output leaves the split range, or NULL */
  int32_t max_ctas;         /* grid = min(tiles, SMs, max_ctas); 0: min(tiles, SMs) as the library's own launches */
  int32_t backend;          /* 0 the wgmma core, 1 the SIMT fp32 FFMA cross-check (epi 0 without converter or identity only) */
} opb_debug_gemm_desc;
int opb_debug_gemm(const opb_debug_gemm_desc* desc, void* stream);
/* The fp16 linear-attention state kernel on a caller-supplied plane kvh [frames*(n_pad+m_pad), 512] (pad rows must be
 * zero); slabs_per_group = 0: the library's own choice; *n_groups = number of partial states; partial [n_groups][4][64*64+64]
 * (NULL: size query only). */
int opb_debug_kv_state_h(const void* kvh, int32_t frames, int32_t n, int32_t m_pts, int32_t slabs_per_group, float* partial,
                         int32_t* n_groups, void* stream);
/* fp32 [rows, cols] -> fp16-split planes: hi = fp16(64 x), lo = fp16(64 x - hi). */
int opb_debug_split(const float* x, void* hi, void* lo, size_t n, void* stream);
/* The block-wide primitives of csrc/block.cuh on their own: one block of `threads` threads (a multiple of 32 in [32, 1024])
 * walks `tiles` consecutive tiles of `threads` inputs `in` and calls one primitive per tile, always with the same shared
 * scratch.  prim 0 block_reduce, 1 block_scan (exclusive; reverse = 1: from the last thread), 2 block_rank (`in` as int32
 * keep flags, nonzero = keep; op 0 only).  op picks the operator and the element type: 0 Sum32, 1 Max, 2 Min (int32),
 * 3 Sum64 (uint64, wrapping), 4 SumS64 (int64).  value and total [tiles][threads] get, per thread and tile, what that thread
 * got: the reduction (in both), the exclusive prefix and the scan's total, or the rank and the block's count. */
int opb_debug_block(int32_t prim, int32_t op, int32_t reverse, int32_t threads, int32_t tiles, const void* in, void* value, void* total,
                    void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ONEPOSE_B200_H_ */
