/* se2gpu — C ABI of the H100-native hot paths of se2lam (ORB front-end, SE(2)-XYZ local BA).
 *
 * Plain C, plain pointers and sizes, int status codes, no exceptions across the boundary.
 * The reference (izhengfan/se2lam) has no FFI layer of its own: the seam is the C++ symbols
 * listed below, which the header shims in include/se2lam/ forward to these entry points
 * (INTEGRATION.md shows the binding).  Every function is implemented by hand-written sm_90a
 * CUDA in se2lam_b200/csrc; there is no CPU fallback — a call without a usable CUDA device
 * returns SE2GPU_ERR_NO_DEVICE.
 *
 *   entry point                      replaces (reference file:line)
 *   -------------------------------  -------------------------------------------------------------
 *   se2gpu_orb_create[_scored]       se2lam::ORBextractor::ORBextractor       src/ORBextractor.cpp:463-520
 *   se2gpu_orb_extract[_device]      se2lam::ORBextractor::operator()         src/ORBextractor.cpp:727-788
 *                                    (ComputePyramid :790-831, ComputeKeyPoints :531-716,
 *                                     IC_Angle :130-157, computeOrbDescriptor :160-200)
 *   se2gpu_hamming_distance          se2lam::ORBmatcher::DescriptorDistance   src/ORBmatcher.cpp:110-126
 *   se2gpu_matcher_create            se2lam::ORBmatcher::ORBmatcher           src/ORBmatcher.cpp:49-51
 *   se2gpu_[matcher_]match_by_window[_device]      ORBmatcher::MatchByWindow  src/ORBmatcher.cpp:278-381
 *                                    (+ Frame grid / GetFeaturesInArea        src/Frame.cpp:64-77, 209-286)
 *   se2gpu_[matcher_]match_by_projection[_device]  ORBmatcher::MatchByProjection  src/ORBmatcher.cpp:383-454
 *   se2gpu_[matcher_]search_by_bow   se2lam::ORBmatcher::SearchByBoW          src/ORBmatcher.cpp:128-276
 *   se2gpu_search_by_bow_batch_device  the same for B keyframe pairs           src/ORBmatcher.cpp:128-276
 *   se2gpu_ba_set_problem            Map::loadLocalGraph -> addVertexSE2 / addEdgeSE2 / addVertexSBAXYZ /
 *                                    addEdgeSE2XYZ / addCamPara               src/Map.cpp:891-1053, src/optimizer.cpp:17-62,207-215,316-324
 *                                    + SparseOptimizer::initializeOptimization(0)   src/LocalMapper.cpp:259
 *   se2gpu_ba_optimize               SlamOptimizer::optimize(Config::LOCAL_ITER)    src/LocalMapper.cpp:260
 *                                    (EdgeSE2XYZ::computeError/linearizeOplus src/EdgeSE2XYZ.cpp:61-106,
 *                                     PreEdgeSE2 include/se2lam/EdgeSE2XYZ.h:62-102, g2o LM/Schur/Cholesky/Huber [upstream])
 *   se2gpu_ba_get[_f32]              estimateVertexSE2 / estimateVertexSBAXYZ src/optimizer.cpp:45-50, 549-554
 *                                    (+ the float write-back of Map::optimizeLocalGraph  src/Map.cpp:768-779)
 *   se2gpu_ba_build_information      per-edge Omega of Map::loadLocalGraph    src/Map.cpp:1024-1049
 *   se2gpu_voc_create / _transform   DBoW2 TemplatedVocabulary::transform     Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1220-1262
 *   se2gpu_voc_compute_bow_device    KeyFrame::ComputeBoW (transform(features, v, fv, levelsup)) src/KeyFrame.cpp:244-254,
 *                                                                             TemplatedVocabulary.h:1150-1216
 *   se2gpu_median_descriptor         MapPoint::updateMainKFandDescriptor      src/MapPoint.cpp:228-272
 *   se2gpu_triangulate[_device]      cvu::triangulate                         src/cvutil.cpp:46-59
 *   se2gpu_track_triangulate[_device]  Track::doTriangulate                   src/Track.cpp:389-416
 *   se2gpu_xyz_info[_device]         Track::calcSE3toXYZInfo                  src/Track.cpp:259-306
 *   se2gpu_projection_observations[_device]  LocalMapper::findCorrespd, MatchByProjection branch  src/LocalMapper.cpp:119-141
 *   se2gpu_mp_add_observations[_device]      MapPoint::addObservation   src/MapPoint.cpp:104-185, 228-292
 *   se2gpu_mp_erase_observations[_device]    MapPoint::eraseObservation src/MapPoint.cpp:86-101
 *   se2gpu_mp_update_measure[_device]        MapPoint::updateMeasureInKFs  src/MapPoint.cpp:294-305 (src/Map.cpp:779-780)
 *   se2gpu_remove_outliers[_device]  Track::removeOutliers (cv::findFundamentalMat)  src/Track.cpp:308-344
 *   se2gpu_pose_ba[_device]          Localizer::DoLocalBA (pose-only SE(3) BA, g2o LM)  src/Localizer.cpp:233-302,
 *                                    (addPlaneMotionSE3Expmap src/optimizer.cpp:236-314, EdgeSE3ExpmapPrior :159-189)
 *   se2gpu_localizer_ba_device       Localizer::MatchLocalMap's observations + DoLocalBA  src/Localizer.cpp:211-302
 *   se2gpu_feat_edge[_device]        GlobalMapper::CreateFeatEdge (both overloads), OptKFPair, OptKFPairMatch
 *                                    src/GlobalMapper.cpp:737-1032 (addVertexSE3PlaneMotion src/optimizer.cpp:337-468),
 *                                    Sparsifier::DoMarginalizeSE3XYZ / InfoSE3  src/sparsifier.cpp:59-274
 *   se2gpu_global_ba[_device]        GlobalMapper::GlobalBA's pose graph and optimize(GLOBAL_ITER)  src/GlobalMapper.cpp:328-504
 *                                    (addVertexSE3PlaneMotion src/optimizer.cpp:337-468, addEdgeSE3 :375-419)
 *   se2gpu_global_ba_update_points[_device]  GlobalBA's map-point write-back  src/GlobalMapper.cpp:506-531
 *   se2gpu_detect_loop_device        GlobalMapper::DetectLoopClose / Localizer::DetectLoopClose (DBoW2 L1Scoring::score)
 *                                    src/GlobalMapper.cpp:201-254, src/Localizer.cpp:337-392,
 *                                    Thirdparty/DBoW2/DBoW2/ScoringObject.cpp:23-68
 *   se2gpu_verify_loop_device        GlobalMapper::VerifyLoopClose / Localizer::VerifyLoopClose  src/GlobalMapper.cpp:256-326,
 *                                    (RemoveMatchOutlierRansac :1207-1248, RemoveKPMatch :1251-1276) src/Localizer.cpp:394-431
 */
#ifndef SE2GPU_H
#define SE2GPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SE2GPU_OK 0
#define SE2GPU_ERR_NO_DEVICE -1
#define SE2GPU_ERR_CUDA -2
#define SE2GPU_ERR_INVALID -3
#define SE2GPU_ERR_CAPACITY -4

/* ------------------------------------------------------------------------------------------ common */
int se2gpu_device_count(void);
/* last error message of the calling thread ("" if none) */
const char* se2gpu_last_error(void);
/* number of kernel launches issued by this library in this process so far (bench.py's gpu_launches) */
unsigned long long se2gpu_launch_count(void);

/* ------------------------------------------------------------------------------------------ ORB */
typedef struct se2gpu_orb se2gpu_orb;

/* bit-identical to cv::KeyPoint (28 bytes) so results can be copied straight into a
 * std::vector<cv::KeyPoint> */
typedef struct se2gpu_keypoint {
    float x, y;      /* pt, in level-0 pixel coordinates */
    float size;      /* PATCH_SIZE * scale(level), truncated to int */
    float angle;     /* degrees, [0,360) */
    float response;  /* FAST score, or Harris response for HARRIS_SCORE handles */
    int octave;      /* pyramid level */
    int class_id;    /* -1 */
} se2gpu_keypoint;

/* ORBextractor(nfeatures, scaleFactor, nlevels, FAST_SCORE, fastTh) for frames up to max_w x max_h,
 * batches of up to max_batch frames, on CUDA device `device`. Returns NULL on failure. */
se2gpu_orb* se2gpu_orb_create(int nfeatures, float scale_factor, int nlevels, int fast_th, int max_w, int max_h,
                              int max_batch, int device);
/* ORBextractor::scoreType values (reference include/se2lam/ORBextractor.h:44) */
#define SE2GPU_ORB_HARRIS_SCORE 0
#define SE2GPU_ORB_FAST_SCORE 1
/* ORBextractor(nfeatures, scaleFactor, nlevels, scoreType, fastTh), the reference constructor's argument order. With
 * HARRIS_SCORE every cell's FAST keypoints are ranked by their Harris response (7x7 block, k = 0.04, on the un-blurred
 * level, ORBextractor.cpp:85-126, :625-629) instead of the FAST score, and keypoint.response is that response. A Harris
 * handle also holds 8 B per candidate slot per frame (about 2 MB per 640x480 frame at 1000 features). Returns NULL with
 * a message for an unknown score type. se2gpu_orb_create(...) == se2gpu_orb_create_scored(..., FAST_SCORE, ...). */
se2gpu_orb* se2gpu_orb_create_scored(int nfeatures, float scale_factor, int nlevels, int score_type, int fast_th, int max_w,
                                     int max_h, int max_batch, int device);
void se2gpu_orb_destroy(se2gpu_orb* h);

/* operator() over a batch of n frames held in HOST memory (CV_8UC1, row stride `stride` bytes, frame i at
 * imgs + i*frame_stride). Synchronous: copies frames in, runs the extractor, copies results out.
 *   kps    [n * nfeatures]      frame i's keypoints start at kps + i*nfeatures
 *   desc   [n * nfeatures * 32] 256-bit rBRIEF, row i*nfeatures + k belongs to kps[i*nfeatures + k]
 *   counts [n]                  number of keypoints of each frame (<= nfeatures)
 * An empty image (w<=0 || h<=0 || imgs==NULL) returns SE2GPU_OK with all counts 0 (the reference returns
 * silently, ORBextractor.cpp:730-731). */
int se2gpu_orb_extract(se2gpu_orb* h, const uint8_t* imgs, int n, int w, int hgt, int stride, size_t frame_stride,
                       se2gpu_keypoint* kps, uint8_t* desc, int* counts);

/* Asynchronous, two-deep form of se2gpu_orb_extract for streams of batches: _submit enqueues the copies and kernels of one
 * batch and returns at once; _wait blocks until the OLDEST submitted batch is complete and its results are in the buffers
 * handed to _submit. Up to two batches may be in flight, so the host->device copy of batch k+1 and the device->host copy of
 * batch k-1 overlap the kernels of batch k (a second internal context is created on first use). The buffers of a submitted
 * batch must stay valid and untouched until its _wait returns; page-locked buffers make the copies true DMA transfers. */
int se2gpu_orb_submit(se2gpu_orb* h, const uint8_t* imgs, int n, int w, int hgt, int stride, size_t frame_stride,
                      se2gpu_keypoint* kps, uint8_t* desc, int* counts);
int se2gpu_orb_wait(se2gpu_orb* h);

/* Same with DEVICE buffers (frames already resident in HBM, results left in HBM); asynchronous on
 * `stream` (a cudaStream_t passed as void*; NULL = the default stream). */
int se2gpu_orb_extract_device(se2gpu_orb* h, const uint8_t* d_imgs, int n, int w, int hgt, int stride,
                              size_t frame_stride, se2gpu_keypoint* d_kps, uint8_t* d_desc, int* d_counts, void* stream);

/* parity/debug: geometry and contents of pyramid level `level` of frame `frame` from the last extract.
 * out must hold (h+32)*pitch bytes where pitch/h come from se2gpu_orb_level_dims. blurred!=0 returns the
 * Gaussian-blurred plane the descriptors were sampled from. */
int se2gpu_orb_level_dims(se2gpu_orb* h, int level, int* w, int* hgt, int* pitch);
int se2gpu_orb_get_level(se2gpu_orb* h, int frame, int level, int blurred, uint8_t* out);

/* per-kernel device timing (CUDA events on the launching stream) for bench.py's roofline line.
 * groups: 0 pyramid (orb_pyr0 + orb_resize_w), 1 FAST (orb_fast_cells or orb_fast_cells_big, plus orb_harris on HARRIS_SCORE
 * handles), 2 orb_select, 3 orb_blur,
 * 4 orb_orient_describe.
 * enable!=0 starts/restarts accumulation; read returns accumulated milliseconds and launch counts per group
 * (synchronises the events it reads). */
#define SE2GPU_ORB_PROFILE_GROUPS 5
int se2gpu_orb_profile(se2gpu_orb* h, int enable);
int se2gpu_orb_profile_read(se2gpu_orb* h, double* ms, int* launches);

/* Folds the lens undistortion that Frame::Frame applies right before the extractor (reference src/Frame.cpp:22:
 * cv::undistort(im, img, Config::Kcam, Config::Dcam)) into the pyramid's level 0: after this call the frames handed to
 * se2gpu_orb_extract / _extract_device are RAW frames and the keypoints/descriptors are those of the undistorted frame,
 * bit-identical to undistort-then-extract. K: 3x3 row-major float32 camera matrix (Config::Kcam), dist: 0/4/5/8/12
 * float32 coefficients (k1 k2 p1 p2 [k3 [k4 k5 k6 [s1 s2 s3 s4]]], Config::Dcam). K == NULL switches it off. */
int se2gpu_orb_set_undistort(se2gpu_orb* h, const float* K, const float* dist, int ndist);
/* Test hook (host only, no GPU needed): the fixed-point map se2gpu_orb_set_undistort builds for a w x h frame;
 * m1 [h*w*2] int16 integer source coordinates (x, y), m2 [h*w] uint16 fraction index (fy*32 + fx). */
int se2gpu_orb_debug_undistort_map(const float* K, const float* dist, int ndist, int w, int h, int16_t* m1, uint16_t* m2);

/* Test hook for the device selection primitive behind KeyPointsFilter::retainBest (ORBextractor.cpp:692, :708):
 * runs the warp-cooperative std::nth_element on `count` independent lists of packed records (score in bits 31..24)
 * stored back to back in HOST memory; list k is values[offsets[k] .. offsets[k+1]) and is permuted in place exactly
 * as std::nth_element(begin, begin + nth[k], end, score-greater) of libstdc++ would. */
int se2gpu_orb_debug_nth_element(uint32_t* values, const int* offsets, const int* nth, int count, int device);
/* The same for the Harris-score selection: float responses (no NaN) in HOST memory, list k = values[offsets[k] ..
 * offsets[k+1]); perm receives, for every position of list k, the list-local index of the element that
 * std::nth_element(begin, begin + nth[k], end, response-greater) of libstdc++ leaves there. */
int se2gpu_orb_debug_nth_element_f32(const float* values, const int* offsets, const int* nth, int count, int* perm, int device);

/* ------------------------------------------------------------------------------------------ matcher */
/* DescriptorDistance for n pairs of 32-byte descriptors in HOST memory: out[i] = popcount(a_i ^ b_i) */
int se2gpu_hamming_distance(const uint8_t* a, const uint8_t* b, int n, int* out, int device);

/* Keypoint grid of Frame (64 x 48 cells over [minX,maxX) x [minY,maxY)): inv_w = 64/(maxX-minX) etc. */
typedef struct se2gpu_grid_params {
    float min_x, min_y, inv_w, inv_h;
} se2gpu_grid_params;

/* Matcher context: owns every device buffer the matchers need for up to max_queries query items (frame-1 keypoints / map
 * points / KF1 features) against up to max_db database keypoints (candidate table max_queries x max_db x 8 bytes), a
 * stream and page-locked staging for the host entry points. No allocation happens per call. One context per calling
 * thread (like the reference's stack-allocated ORBmatcher objects, the calls are not re-entrant on one context). */
typedef struct se2gpu_matcher se2gpu_matcher;
se2gpu_matcher* se2gpu_matcher_create(int max_queries, int max_db, int device);
/* The same for the batched device entry points below, up to max_batch (<= 65535) frame pairs per call: the candidate table
 * becomes max_batch x max_queries x max_db x 8 bytes (at most 4 GiB in all) and every pair gets its own scratch.
 * se2gpu_matcher_create(q, d, dev) == se2gpu_matcher_create_batch(q, d, 1, dev). */
se2gpu_matcher* se2gpu_matcher_create_batch(int max_queries, int max_db, int max_batch, int device);
void se2gpu_matcher_destroy(se2gpu_matcher* m);

/* MatchByWindow(frame1, frame2, vbPrevMatched, winSize, vnMatches12, levelOffset, minLevel, maxLevel) with nnratio =
 * ORBmatcher::mfNNratio on DEVICE buffers, asynchronous on `stream` (cudaStream_t as void*, NULL = default stream): the
 * keypoint / descriptor buffers are the ones se2gpu_orb_extract_device wrote (reference call chain Track.cpp:129-132 runs
 * the extractor and MatchByWindow back to back), nothing crosses PCIe. n1 / n2 are capacities; d_n1 / d_n2 (may be NULL)
 * point to the actual counts in device memory (e.g. the extractor's d_counts entries). d_prev [n1*2] is vbPrevMatched,
 * updated in place; d_matches12 [n1]; d_nmatches (may be NULL) receives the match count. */
int se2gpu_match_by_window_device(se2gpu_matcher* m, const se2gpu_keypoint* d_kp1, const uint8_t* d_desc1, int n1, const int* d_n1,
                                  const se2gpu_keypoint* d_kp2, const uint8_t* d_desc2, int n2, const int* d_n2, float* d_prev,
                                  se2gpu_grid_params grid, int win_size, int level_offset, int min_level, int max_level,
                                  float nnratio, int* d_matches12, int* d_nmatches, void* stream);
/* vbPrevMatched initialisation (Track.cpp:113-116: the reference frame's keypoint positions): d_xy[2i..] = d_kp[i].pt */
int se2gpu_keypoints_to_points_device(const se2gpu_keypoint* d_kp, int n, const int* d_n, float* d_xy, void* stream);

/* MatchByProjection on DEVICE buffers (same flattening of the object graph as se2gpu_match_by_projection below). */
int se2gpu_match_by_projection_device(se2gpu_matcher* m, const se2gpu_keypoint* d_kf_kp, const uint8_t* d_kf_desc, int n_kf,
                                      const int* d_n_kf, const uint8_t* d_kf_observed, const uint8_t* d_mp_valid,
                                      const float* d_mp_uv, int n_mp, const int* d_mp_octave, const uint8_t* d_mp_desc,
                                      se2gpu_grid_params grid, int win_size, int level_offset, float nnratio,
                                      int* d_matches_idx_mp, int* d_nmatches, void* stream);

/* The two device entry points over a batch of B independent frame pairs in one call, with the extractor's layout (frame i
 * at d_kps + i*nfeatures): pair b reads d_kp1 + b*cap1, d_desc1 + b*cap1*32, d_kp2 + b*cap2, d_desc2 + b*cap2*32 and
 * the counts d_n1[b], d_n2[b] (either array may be NULL: every pair at its capacity), updates d_prev + b*cap1*2 and
 * writes d_matches12 + b*cap1 and d_nmatches[b] (may be NULL) - so d_matches12 feeds se2gpu_remove_outliers_device as is.
 * Pair b's outputs are the bytes the single-pair call makes for that pair alone with n1 = cap1, n2 = cap2 (matches,
 * vbPrevMatched, match count, and the rounds / fallback flag of se2gpu_matcher_last_rounds_batch). All pairs share one
 * grid: the reference's Frame grid bounds are static members, the same for every frame. The kernel launches are those of
 * one single-pair call whatever B is. B > max_batch, cap1 > max_queries or cap2 > max_db: SE2GPU_ERR_CAPACITY; B < 0 or
 * a NULL required pointer: SE2GPU_ERR_INVALID; B == 0 does nothing. */
int se2gpu_match_by_window_batch_device(se2gpu_matcher* m, int B, const se2gpu_keypoint* d_kp1, const uint8_t* d_desc1, int cap1,
                                        const int* d_n1, const se2gpu_keypoint* d_kp2, const uint8_t* d_desc2, int cap2,
                                        const int* d_n2, float* d_prev, se2gpu_grid_params grid, int win_size, int level_offset,
                                        int min_level, int max_level, float nnratio, int* d_matches12, int* d_nmatches,
                                        void* stream);
/* MatchByProjection for B (keyframe, map-point list) pairs: keyframe side as frame 2 above (d_kf_kp + b*cap_kf, d_kf_desc +
 * b*cap_kf*32, d_n_kf[b], d_kf_observed + b*cap_kf, d_matches_idx_mp + b*cap_kf, d_nmatches[b]); map points in slots of
 * cap_mp (d_mp_valid / d_mp_octave + b*cap_mp, d_mp_uv + b*cap_mp*2, d_mp_desc + b*cap_mp*32). A pair with fewer map
 * points pads its slot with mp_valid = 0: the reference skips such a point (ORBmatcher.cpp:390-404) and the padding comes
 * after every real one, so the result is that of the shorter list. */
int se2gpu_match_by_projection_batch_device(se2gpu_matcher* m, int B, const se2gpu_keypoint* d_kf_kp, const uint8_t* d_kf_desc,
                                            int cap_kf, const int* d_n_kf, const uint8_t* d_kf_observed,
                                            const uint8_t* d_mp_valid, const float* d_mp_uv, int cap_mp, const int* d_mp_octave,
                                            const uint8_t* d_mp_desc, se2gpu_grid_params grid, int win_size, int level_offset,
                                            float nnratio, int* d_matches_idx_mp, int* d_nmatches, void* stream);

/* HOST-buffer entry points on an explicit context (synchronous; one stream synchronisation per call).
 * MatchByWindow: prev [n1*2] is vbPrevMatched, updated in place. matches12 [n1]. Returns the number of matches (>=0)
 * or a negative error. */
int se2gpu_matcher_match_by_window(se2gpu_matcher* m, const se2gpu_keypoint* kp1, const uint8_t* desc1, int n1,
                                   const se2gpu_keypoint* kp2, const uint8_t* desc2, int n2, float* prev,
                                   se2gpu_grid_params grid, int win_size, int level_offset, int min_level, int max_level,
                                   float nnratio, int* matches12);
/* MatchByProjection(pNewKF, localMPs, winSize, levelOffset, vMatchesIdxMP), object graph flattened:
 *   mp_valid[i]  = !isNull && isGoodPrl && !pNewKF->hasObservation(pMP) && inImgBound(predictUV)
 *   mp_uv[i]     = predictUV;  mp_octave[i] = mMainOctave;  mp_desc = mMainDescriptor
 *   kf_observed[k] = pNewKF->hasObservation(k)
 * matches_idx_mp [n_kf]. Returns the number of matches. */
int se2gpu_matcher_match_by_projection(se2gpu_matcher* m, const se2gpu_keypoint* kf_kp, const uint8_t* kf_desc, int n_kf,
                                       const uint8_t* kf_observed, const uint8_t* mp_valid, const float* mp_uv, int n_mp,
                                       const int* mp_octave, const uint8_t* mp_desc, se2gpu_grid_params grid, int win_size,
                                       int level_offset, float nnratio, int* matches_idx_mp);
/* SearchByBoW(pKF1, pKF2, mapMatches12, bIfMPOnly); each DBoW2::FeatureVector flattened to ascending node
 * ids + CSR feature lists (ptr has n_node+1 entries). matches12 [n1], -1 = unmatched. */
typedef struct se2gpu_bow_kf {
    const float* angle;     /* keyPointsUn[i].angle */
    const uint8_t* desc;    /* [n*32] */
    const uint8_t* has_mp;  /* GetMapPointMatches()[i] && !isNull */
    int n;
    const int* node;        /* ascending node ids */
    int n_node;
    const int* ptr;         /* [n_node+1] */
    const int* feat;        /* feature indices */
} se2gpu_bow_kf;
int se2gpu_matcher_search_by_bow(se2gpu_matcher* m, const se2gpu_bow_kf* kf1, const se2gpu_bow_kf* kf2, int mp_only,
                                 float nnratio, int check_orientation, int* matches12);

/* SearchByBoW (src/ORBmatcher.cpp:128-276) for B keyframe pairs on DEVICE buffers, asynchronous on `stream`. One side of
 * the batch: keyframe k's features in slot k of `cap` entries, its FeatureVector exactly as se2gpu_voc_compute_bow_device
 * writes it (node + k*cap ascending, ptr + k*(cap+1), feat + k*cap, n_node[k]). */
typedef struct se2gpu_bow_batch_kf {
    const se2gpu_keypoint* kp;  /* [slots*cap] keyPointsUn; the angle is read */
    const uint8_t* desc;        /* [slots*cap*32] */
    const uint8_t* has_mp;      /* [slots*cap] GetMapPointMatches()[i] && !isNull; may be NULL when mp_only == 0 */
    int cap;                    /* features per slot */
    const int* node;            /* [slots*cap] ascending node ids, n_node[k] of them */
    const int* ptr;             /* [slots*(cap+1)] */
    const int* feat;            /* [slots*cap] feature indices of each node, ascending */
    const int* n_node;          /* [slots] */
} se2gpu_bow_batch_kf;
/* Pair b matches keyframe b of kf1 against keyframe d_slot2[b] of kf2 (d_slot2 NULL: keyframe b), so that a map's
 * keyframes assembled once can be matched against many frames without copies. Writes d_matches12 + b*kf1->cap (-1 =
 * unmatched) and d_nmatches[b] (may be NULL). Pair b's result is that of se2gpu_matcher_search_by_bow on the same two
 * keyframes. The launches - the node walk (k_bow_walk, one CTA per pair), the candidates, the resolve and the sequential
 * fallback; the resolve is left out when its claim table does not fit in shared memory - are the same whatever B is. Capacities are checked on the host: B > max_batch, kf1->cap > max_queries or
 * kf2->cap > max_db is SE2GPU_ERR_CAPACITY (a pair has at most kf1->cap queries and a node list at most kf2->cap items).
 * B < 0, a negative cap or a NULL required pointer is SE2GPU_ERR_INVALID; B == 0 does nothing. Like every device entry,
 * it trusts the contents of device memory: the FeatureVectors must be well formed (ascending, unrepeated node ids, ptr
 * ascending within [0, cap], feature indices below cap, each feature in at most one node) and every d_slot2[b] a slot of
 * kf2's arrays or negative. A negative d_slot2[b] makes pair b empty: no queries, d_matches12 + b*kf1->cap all -1,
 * d_nmatches[b] = 0, and nothing of kf2 is read for it. Calls on one context are ordered like the other device entries (its scratch is shared). */
int se2gpu_search_by_bow_batch_device(se2gpu_matcher* m, int B, const se2gpu_bow_batch_kf* kf1, const se2gpu_bow_batch_kf* kf2,
                                      const int* d_slot2, int mp_only, float nnratio, int check_orientation, int* d_matches12,
                                      int* d_nmatches, void* stream);

/* The same three with a context per device created on first use and kept for the life of the process. */
int se2gpu_match_by_window(const se2gpu_keypoint* kp1, const uint8_t* desc1, int n1, const se2gpu_keypoint* kp2,
                           const uint8_t* desc2, int n2, float* prev, se2gpu_grid_params grid, int win_size,
                           int level_offset, int min_level, int max_level, float nnratio, int* matches12, int device);
int se2gpu_match_by_projection(const se2gpu_keypoint* kf_kp, const uint8_t* kf_desc, int n_kf,
                               const uint8_t* kf_observed, const uint8_t* mp_valid, const float* mp_uv, int n_mp,
                               const int* mp_octave, const uint8_t* mp_desc, se2gpu_grid_params grid, int win_size,
                               int level_offset, float nnratio, int* matches_idx_mp, int device);
int se2gpu_search_by_bow(const se2gpu_bow_kf* kf1, const se2gpu_bow_kf* kf2, int mp_only, float nnratio,
                         int check_orientation, int* matches12, int device);

/* per-kernel device timing for bench.py; groups: 0 k_grid_build, 1 k_candidates, 2 k_resolve, 3 k_fallback_* */
#define SE2GPU_MATCHER_PROFILE_GROUPS 4
int se2gpu_matcher_profile(se2gpu_matcher* m, int enable);
int se2gpu_matcher_profile_read(se2gpu_matcher* m, double* ms, int* launches);
/* diagnostics of the last resolve on this context: speculative rounds it took, and whether the sequential fallback ran */
int se2gpu_matcher_last_rounds(se2gpu_matcher* m, int* rounds, int* used_fallback);
/* the same for every pair of the last batched call: rounds [B], used_fallback [B] (either may be NULL); B larger than
 * that call's batch is SE2GPU_ERR_INVALID */
int se2gpu_matcher_last_rounds_batch(se2gpu_matcher* m, int B, int* rounds, int* used_fallback);

/* ------------------------------------------------------------------------------------------ bag of words */
/* DBoW2 vocabulary tree (TemplatedVocabulary<FORB::TDescriptor, FORB>, reference Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h)
 * flattened: node 0 is the root (m_nodes[0]); node i has the 32-byte descriptor node_desc[32 i], the children
 * children[child_ptr[i] .. child_ptr[i+1]) in m_nodes[i].children order, and - for a leaf - word_id[i] >= 0 and its weight
 * (inner nodes: word_id -1). levels = m_L. */
typedef struct se2gpu_voc se2gpu_voc;
se2gpu_voc* se2gpu_voc_create(int n_nodes, const uint8_t* node_desc, const int* child_ptr, const int* children,
                              const int* word_id, const double* weight, int levels, int device);
void se2gpu_voc_destroy(se2gpu_voc* v);
/* transform(feature, word_id, weight, &nid, levelsup) (TemplatedVocabulary.h:1220-1262) for n descriptors [n*32]:
 * word_id [n], weight [n], node_id [n] (may be NULL) = the node at level m_L - levelsup on the feature's path (0 = root
 * when that level is <= 0; -1 when the leaf is shallower - the reference leaves *nid unset there). This host entry leaves
 * the BowVector / FeatureVector assembly of transform(features, v, fv, levelsup) (:1150-1216: v.addWeight(id, w) in
 * feature order, fv.addFeature(nid, i), L1 normalisation) to the caller; se2gpu_voc_compute_bow_device below does it on
 * the device. KeyFrame::ComputeBoW (src/KeyFrame.cpp:244-254) uses levelsup = 4. HOST buffers, synchronous. */
int se2gpu_voc_transform(se2gpu_voc* v, const uint8_t* desc, int n, int levelsup, int* word_id, double* weight, int* node_id);
/* same on DEVICE buffers (e.g. the extractor's d_desc), asynchronous on `stream` */
int se2gpu_voc_transform_device(se2gpu_voc* v, const uint8_t* d_desc, int n, int levelsup, int* d_word_id, double* d_weight,
                                int* d_node_id, void* stream);
/* KeyFrame::ComputeBoW (src/KeyFrame.cpp:244-254) for B keyframes: transform(features, v, fv, levelsup)
 * (TemplatedVocabulary.h:1150-1216) with TF_IDF weighting and L1 normalisation, the ORBvoc settings, on DEVICE buffers,
 * asynchronous on `stream`. Keyframe b's descriptors are d_desc + b*cap*32, d_n[b] of them (d_n NULL: cap). Keyframe b's
 * outputs, all strided by cap:
 *   BowVector      d_bow_word + b*cap ascending word ids, d_bow_value + b*cap their values, d_bow_n[b] words;
 *   FeatureVector  d_fv_node + b*cap ascending node ids, d_fv_ptr + b*(cap+1) (ptr[0] = 0, ptr[n_node] = features used),
 *                  d_fv_feat + b*cap the feature indices of each node, ascending, d_fv_n[b] nodes.
 * The three BowVector outputs are all NULL when only the FeatureVector is wanted. Entries past the counts are unspecified.
 * Bit-identical to DBoW2: a feature takes part only when its weight is > 0 (:1181); a word's value is the double sum of
 * its features' weights in ascending feature order; the L1 norm is the sum of |value| in ascending word order, and the
 * values are divided by it when it is > 0 (BowVector.cpp:62-84). Node -1 (the leaf is shallower than level m_L - levelsup;
 * the reference leaves the node id unset there) is kept as a node like any other and sorts first.
 * Two launches whatever B is (the descent over B*cap slots, the assembly with one CTA per keyframe). The descent's triples
 * live in scratch of the vocabulary handle, which grows only when a call needs more than any earlier one: calls on one
 * handle are ordered (one stream or host-synchronised), and a call no larger than an earlier one allocates nothing, does
 * not synchronise the host and may be captured in a CUDA graph. cap above the assembly's shared memory (36 bytes per
 * feature: 6 400 features on an H100) is SE2GPU_ERR_CAPACITY; B < 0, cap < 0, some but not all BowVector outputs NULL or
 * a NULL FeatureVector output is SE2GPU_ERR_INVALID; B == 0 does nothing. */
int se2gpu_voc_compute_bow_device(se2gpu_voc* v, int B, const uint8_t* d_desc, int cap, const int* d_n, int levelsup, int* d_bow_word,
                                  double* d_bow_value, int* d_bow_n, int* d_fv_node, int* d_fv_ptr, int* d_fv_feat, int* d_fv_n,
                                  void* stream);

/* MapPoint::updateMainKFandDescriptor (reference src/MapPoint.cpp:228-272) for M map points at once: the descriptors of map
 * point m's observations are desc rows ptr[m] .. ptr[m+1]); best_idx [m] = index (within the point's list) of the descriptor
 * with the least median Hamming distance to the others - median = element int(0.5*(N-1)) of the sorted distances incl. the
 * zero self-distance, first index wins ties - and best_median [m] (may be NULL) that median. HOST buffers. */
int se2gpu_median_descriptor(const uint8_t* desc, const int* ptr, int M, int* best_idx, int* best_median, int device);

/* ------------------------------------------------------------------------------------------ two-view geometry */
/* Reproduces the reference's float arithmetic and OpenCV's primitives on an x86-64 AVX2 host with glibc 2.39 bit for bit, with
 * two steps matched by restatement rather than proven against cv2 (DESIGN.md section 8): the double hypot inside the SVD
 * (OpenCV's lapack.cpp template, which cv2 does not expose) and the last bits of sin/cos inside Rodrigues (the device's
 * sincos is not glibc's; a difference survives the rounding to float only at a float rounding boundary). NaN results
 * are NaN on both sides with possibly different payloads.
 * Projection matrices are 3x4 row-major floats (Config::Kcam * Tcw.rowRange(0,3)); poses are 4x4 row-major floats.
 * The _device forms take DEVICE buffers and are asynchronous on `stream` (cudaStream_t as void*, NULL = default stream);
 * the others take HOST buffers, run on `device` and return when the results are in place. */

/* cvu::triangulate (src/cvutil.cpp:46-59) for n pairs: xyz[3i..] = triangulate(pt1[i], pt2[i], P[idx1[i]], P[idx2[i]]),
 * pt1/pt2 [n*2], P [n_proj*12]. NaN / inf results (w = 0) are returned as computed. */
int se2gpu_triangulate(int n, const float* pt1, const float* pt2, const float* P, int n_proj, const int* idx1, const int* idx2,
                       float* xyz, int device);
int se2gpu_triangulate_device(int n, const float* d_pt1, const float* d_pt2, const float* d_P, const int* d_idx1,
                              const int* d_idx2, float* d_xyz, void* stream);

/* Track::doTriangulate (src/Track.cpp:389-416) after its nMinFrames early return, which stays with the caller. kp_kf [n_kf]
 * are the reference keyframe's keyPointsUn, kp_frame the current frame's, matches12 [n_kf] the result of MatchByWindow
 * (updated in place: -1 where the depth test fails), kf_observed [n_kf] mpKF->hasObservation(i), kf_view_mp [n_kf*3]
 * mpKF->mViewMPs, Tcr [16] mFrame.Tcr, K [9] Config::Kcam, lower/upper_depth Config::LOWER/UPPER_DEPTH,
 * min_parallax_deg the checkParallax degree (1..4; the reference uses 2). local_mps [n_kf*3] is updated in place: unmatched
 * entries and those failing the depth test keep their previous value. good_prl [n_kf] = mvbGoodPrl,
 * counts [2] = {nTrackedOld, nGoodPrl}. The _device form takes d_n_kf (may be NULL) with the keyframe's keypoint count
 * (<= n_kf) as the extractor wrote it; entries at or past it are not touched. */
int se2gpu_track_triangulate(const se2gpu_keypoint* kp_kf, int n_kf, const se2gpu_keypoint* kp_frame, int n_frame, int* matches12,
                             const uint8_t* kf_observed, const float* kf_view_mp, const float* Tcr, const float* K,
                             float lower_depth, float upper_depth, int min_parallax_deg, float* local_mps, uint8_t* good_prl,
                             int* counts, int device);
int se2gpu_track_triangulate_device(const se2gpu_keypoint* d_kp_kf, int n_kf, const int* d_n_kf, const se2gpu_keypoint* d_kp_frame,
                                    int* d_matches12, const uint8_t* d_kf_observed, const float* d_kf_view_mp, const float* d_Tcr,
                                    const float* d_K, float lower_depth, float upper_depth, int min_parallax_deg,
                                    float* d_local_mps, uint8_t* d_good_prl, int* d_counts, void* stream);

/* The same for B independent streams in one launch: stream b reads d_kp_kf + b*cap (d_n[b] keypoints, d_n may be NULL: cap),
 * d_kp_frame + b*cap_frame, d_kf_observed + b*cap, d_kf_view_mp + 3*b*cap and d_Tcr + 16*b, and updates d_matches12 + b*cap,
 * d_local_mps + 3*b*cap, d_good_prl + b*cap and d_counts[2b], d_counts[2b+1]. d_gate [B] (may be NULL: every stream runs) is
 * the nMinFrames test: a stream with d_gate[b] == 0 returns at once and leaves its matches, local map points and flags as
 * they were (its counts are 0). Stream b's outputs are the bytes se2gpu_track_triangulate_device makes for it alone;
 * that call is this one with B = 1. B > 65535: SE2GPU_ERR_CAPACITY. */
int se2gpu_track_triangulate_batch_device(int B, const se2gpu_keypoint* d_kp_kf, int cap, const int* d_n, const se2gpu_keypoint* d_kp_frame,
                                          int cap_frame, int* d_matches12, const uint8_t* d_kf_observed, const float* d_kf_view_mp,
                                          const float* d_Tcr, const int* d_gate, const float* d_K, float lower_depth,
                                          float upper_depth, int min_parallax_deg, float* d_local_mps, uint8_t* d_good_prl,
                                          int* d_counts, void* stream);

/* Track::calcSE3toXYZInfo (src/Track.cpp:259-306) for n points: calcSE3toXYZInfo(xyz1[i], Tcw[pose1[i]], Tcw[pose2[i]]),
 * Tcw [n_pose*16], fx = Config::fxCam. info1/info2 [n*9] are the float matrices widened to double (toMatrix3d). */
int se2gpu_xyz_info(int n, const float* xyz1, const int* pose1, const int* pose2, const float* Tcw, int n_pose, float fx,
                    double* info1, double* info2, int device);
int se2gpu_xyz_info_device(int n, const float* d_xyz1, const int* d_pose1, const int* d_pose2, const float* d_Tcw, float fx,
                           double* d_info1, double* d_info2, void* stream);

/* Body of LocalMapper::findCorrespd's MatchByProjection loop (src/LocalMapper.cpp:119-141) without the object-graph updates.
 * kf_kp [n_kf] are mNewKF->keyPointsUn: their x, y feed the triangulation (keyPointsUn[i].pt) and their octave stands for
 * keyPoints[i].octave, which the undistortion leaves unchanged. matches_idx_mp [n_kf] is the result of MatchByProjection,
 * Tcw_new [16] mNewKF->Tcw.
 * Map point m: mp_main_measure [2m..] getMainMeasure(), mp_main_pose [m] index of mMainKF->Tcw in Tcw_table [n_pose*16],
 * mp_main_octave [m] the main keyframe's octave of the point, mp_normal [3m..] mNormalVector, mp_min_dist / mp_max_dist [m].
 * accept [i] = 1 where the reference adds the observation (acceptNewObserve and the depth window pass); there
 * pos_new_kf [3i..] = posNewKF and info_new [9i..] = infoNew. Rows with accept[i] = 0 are not written. */
int se2gpu_projection_observations(const se2gpu_keypoint* kf_kp, int n_kf, const int* matches_idx_mp, const float* Tcw_new,
                                   const float* mp_main_measure, const int* mp_main_pose, const int* mp_main_octave,
                                   const float* mp_normal, const float* mp_min_dist, const float* mp_max_dist, int n_mp,
                                   const float* Tcw_table, int n_pose, const float* K, float lower_depth, float upper_depth,
                                   float fx, uint8_t* accept, float* pos_new_kf, double* info_new, int device);
int se2gpu_projection_observations_device(const se2gpu_keypoint* d_kf_kp, int n_kf, const int* d_n_kf, const int* d_matches_idx_mp,
                                          const float* d_Tcw_new, const float* d_mp_main_measure, const int* d_mp_main_pose,
                                          const int* d_mp_main_octave, const float* d_mp_normal, const float* d_mp_min_dist,
                                          const float* d_mp_max_dist, const float* d_Tcw_table, const float* d_K, float lower_depth,
                                          float upper_depth, float fx, uint8_t* d_accept, float* d_pos_new_kf, double* d_info_new,
                                          void* stream);

/* ------------------------------------------------------------------------------------------ map-point updates */
/* MapPoint::addObservation (src/MapPoint.cpp:104-122, with updateMainKFandDescriptor :228-292 and updateParallax :124-185),
 * MapPoint::eraseObservation (:86-101) and MapPoint::updateMeasureInKFs (:294-305) over many map points in one call,
 * on the object graph flattened into the tables below (DESIGN.md section 13). Map points are independent: a point's
 * updates touch its own table entries and the keyframe slots of its own observations only. The keyframe side
 * (KeyFrame::addObservation / eraseObservation, and the erasure setNull makes there) is the caller's. */
typedef struct se2gpu_mp_keyframes {
    int n_kf;                    /* K */
    const int* kf_id;            /* [K] mIdKF */
    const uint8_t* kf_null;      /* [K] isNull() */
    const float* Tcw;            /* [K*16] getPose(), row-major */
    const int* kp_base;          /* [K] slot of each keyframe's keypoint 0 */
    int n_slots;                 /* S */
    const se2gpu_keypoint* kp;   /* [S] keyPointsUn[i].pt with keyPoints[i].octave */
    const uint8_t* desc;         /* [S*32] descriptors */
    float* view_mp;              /* [S*3] mViewMPs, in/out */
    double* view_info;           /* [S*9] mViewMPsInfo, in/out */
} se2gpu_mp_keyframes;

/* The point table, in the layout se2gpu_match_by_projection_device (mp_desc, mp_octave) and
 * se2gpu_projection_observations_device (mp_main_measure, mp_main_pose = main_kf, mp_main_octave, mp_normal, mp_min_dist,
 * mp_max_dist) read. Point m observes obs_ptr[m] .. obs_ptr[m+1]-1 (obs_ptr[0] = 0): keyframe obs_kf[j], keypoint
 * obs_idx[j] (slot kp_base[obs_kf[j]] + obs_idx[j]), in mObservations' own iteration order. */
typedef struct se2gpu_mp_points {
    int n_mp;                    /* M */
    float* pos;                  /* [M*3] mPos */
    uint8_t* good_prl;           /* [M] mbGoodParallax */
    uint8_t* null;               /* [M] mbNull */
    int* main_kf;                /* [M] keyframe index of mMainKF, -1 = NULL */
    uint8_t* main_desc;          /* [M*32] mMainDescriptor */
    int* main_octave;            /* [M] mMainOctave */
    float* main_measure;         /* [M*2] getMainMeasure() */
    float* level_scale;          /* [M] mLevelScaleFactor */
    float* normal;               /* [M*3] mNormalVector */
    float* min_dist;             /* [M] mMinDist */
    float* max_dist;             /* [M] mMaxDist */
    const int* obs_ptr;          /* [M+1] */
    const int* obs_kf;           /* [obs_ptr[M]] */
    const int* obs_idx;          /* [obs_ptr[M]] */
} se2gpu_mp_points;

#define SE2GPU_MP_MAX_LEVELS 32
typedef struct se2gpu_mp_params {
    float K[9];                  /* Config::Kcam, row-major */
    float lower_depth, upper_depth; /* Config::LOWER_DEPTH / UPPER_DEPTH */
    float fx;                    /* Config::fxCam */
    int nlevels;                 /* mnScaleLevels, 1 .. SE2GPU_MP_MAX_LEVELS */
    float scale_factors[SE2GPU_MP_MAX_LEVELS]; /* mvScaleFactors */
} se2gpu_mp_params;

/* addObservation for the updates of every point: point m inserts the entries at list positions upd_pos[upd_ptr[m]] ..
 * upd_pos[upd_ptr[m+1]-1], in that order (upd_ptr [M+1], upd_ptr[0] = 0). A point's list is its list AFTER all of its
 * insertions: while one update runs, the entries of its later updates are absent. Each update runs
 * updateMainKFandDescriptor (null keyframes skipped; mMainOctave, mLevelScaleFactor and min/max distances kept when the main
 * keyframe's mIdKF is unchanged), updateParallax (re-triangulation from the oldest observer within 6 keyframe ids, rewriting
 * view_mp / view_info of every observer on success), the mNormalVector update and the final mbNull = false. abandoned [M]
 * is set to 1 for a point updateParallax abandons (setNull) and to 0 otherwise; a later update of that point starts from
 * an empty list. HOST buffers, synchronous; SE2GPU_ERR_INVALID, with nothing changed, for an index outside its table, an
 * update position outside its point's list or repeated within it, or an octave outside nlevels. */
int se2gpu_mp_add_observations(const se2gpu_mp_keyframes* kf, const se2gpu_mp_points* mp, const int* upd_ptr, const int* upd_pos,
                               const se2gpu_mp_params* params, uint8_t* abandoned, int device);
/* eraseObservation: the list given is the list BEFORE the call; the entry at upd_pos is absent once its update has run.
 * A non-null point whose list becomes empty is setNull and reported in abandoned [M]; otherwise
 * updateMainKFandDescriptor and the mNormalVector downdate run. Same rules as above. */
int se2gpu_mp_erase_observations(const se2gpu_mp_keyframes* kf, const se2gpu_mp_points* mp, const int* upd_ptr, const int* upd_pos,
                                 const se2gpu_mp_params* params, uint8_t* abandoned, int device);
/* updateMeasureInKFs for the n points points[0 .. n-1] (after setPos: pos holds se2gpu_ba_get_f32's points):
 * view_mp[slot] = se3map(Tcw, pos) for every observer that is not null. */
int se2gpu_mp_update_measure(const se2gpu_mp_keyframes* kf, const se2gpu_mp_points* mp, int n, const int* points, int device);
/* The same on DEVICE buffers (the structs are host memory holding device pointers), asynchronous on `stream`. The
 * input is checked on the device first: d_status [1] receives SE2GPU_OK, or SE2GPU_ERR_INVALID and then nothing else is
 * written. */
int se2gpu_mp_add_observations_device(const se2gpu_mp_keyframes* kf, const se2gpu_mp_points* mp, const int* d_upd_ptr,
                                      const int* d_upd_pos, const se2gpu_mp_params* params, uint8_t* d_abandoned, int* d_status,
                                      void* stream);
int se2gpu_mp_erase_observations_device(const se2gpu_mp_keyframes* kf, const se2gpu_mp_points* mp, const int* d_upd_ptr,
                                        const int* d_upd_pos, const se2gpu_mp_params* params, uint8_t* d_abandoned,
                                        int* d_status, void* stream);
int se2gpu_mp_update_measure_device(const se2gpu_mp_keyframes* kf, const se2gpu_mp_points* mp, int n, const int* d_points,
                                    int* d_status, void* stream);

/* Test hook: the 4x4 Jacobi SVD behind cvu::triangulate (cv::SVD::compute, MODIFY_A|FULL_UV) on n row-major matrices
 * A [n*16]; w [n*4] singular values (descending), vt [n*16]. HOST buffers. */
int se2gpu_debug_svd4(int n, const float* A, float* w, float* vt, int device);

/* Track::removeOutliers (src/Track.cpp:308-344) for `batch` frame pairs: pt1 / pt2 are the pairs (kp1[i].pt,
 * kp2[matches12[i]].pt) of the matched i in ascending order, mask = cv::findFundamentalMat(pt1, pt2, mask) with OpenCV
 * 4.13's defaults (FM_RANSAC, 3 px, confidence 0.99, 1000 iterations; below 15 pairs OpenCV's LMedS, 7 pairs the 7-point
 * kernel alone, fewer no estimate), matches12[i] = -1 where the mask is 0, then every match -1 when fewer than 10 inliers
 * remain. The RNG, subset draws, epipolar error, acceptance rule and iteration update are OpenCV's bit for bit; the
 * 7-point kernel is this project's own (DESIGN.md section 8).
 * Pair b: kp1 [b*cap1 ..] with n1[b] keypoints (n1 NULL: cap1), kp2 [b*cap2 ..] with n2[b] keypoints, matches12 [b*cap1 ..]
 * updated in place (entries at or past n1[b] untouched), ninliers [b] = the returned nInlier, F [9b ..] (may be NULL) the
 * 3x3 row-major F cv::findFundamentalMat returns (for 7 pairs the first root's), zeros when it returns none, iters [b] (may be
 * NULL) the number of hypotheses the estimator ran. cap1 <= 8192. Host form: matches12 entries must be < n2[b]. */
int se2gpu_remove_outliers(int batch, const se2gpu_keypoint* kp1, const int* n1, int cap1, const se2gpu_keypoint* kp2, const int* n2,
                           int cap2, int* matches12, int* ninliers, double* F, int* iters, int device);
/* Track::removeOutliers (src/Track.cpp:308-344) on DEVICE buffers, asynchronous on `stream`: the extractor's d_kps / d_counts and
 * MatchByWindow's d_matches12 (updated in place), laid out as above; d_n1 / d_n2 may be NULL. A match index at or past
 * the frame-2 count counts as unmatched. */
int se2gpu_remove_outliers_device(int batch, const se2gpu_keypoint* d_kp1, const int* d_n1, int cap1, const se2gpu_keypoint* d_kp2,
                                  const int* d_n2, int cap2, int* d_matches12, int* d_ninliers, double* d_F, int* d_iters,
                                  void* stream);
/* Test hooks of RANSACUpdateNumIters(0.99, ep, 7, max_iters), which the device evaluates through a table built on the host
 * with glibc's log / pow: thresholds [1000] receives the table (the least ep reaching k + 1 iterations; no device needed),
 * and se2gpu_fundam_debug_niters evaluates the device lookup for ep = (n[i] - good[i]) / n[i] (HOST buffers). */
void se2gpu_fundam_niters_table(double* thresholds);
int se2gpu_fundam_debug_niters(int count, const int* n, const int* good, const int* max_iters, int* out, int device);

/* ------------------------------------------------------------------------------------------ loop closure */
/* DetectLoopClose's parameters: a database keyframe with |db_id - q_id| < min_id_offset is not selected
 * (GM_DCL_MIN_KFID_OFFSET), and a loop is detected when the best score is > min_score (GM_DCL_MIN_SCORE_BEST). */
typedef struct se2gpu_loop_detect_params {
    int min_id_offset;
    double min_score;
} se2gpu_loop_detect_params;
#define SE2GPU_LOOP_DETECT_GLOBAL_MAPPER {20, 0.005}  /* src/Config.cpp:80-81 */
#define SE2GPU_LOOP_DETECT_LOCALIZER {0, 0.05}        /* src/Localizer.cpp:341; its current keyframe is not in the map */

/* GlobalMapper::DetectLoopClose (src/GlobalMapper.cpp:201-254) and Localizer::DetectLoopClose (src/Localizer.cpp:337-392)
 * for B query keyframes against N database keyframes, on DEVICE buffers, asynchronous on `stream`, on the current device.
 * BowVectors in the layout se2gpu_voc_compute_bow_device writes: query b's words d_q_word + b*cap_q (ascending), values
 * d_q_value + b*cap_q, d_q_n[b] of them; database keyframe n's at n*cap_db with d_db_n[n]. The database slots are
 * Map::getAllKF()'s order (ascending mIdKF), so that among equal scores the first keyframe wins as in the reference.
 *   d_scores [B*N]  score(q_b, db_n) at b*N + n = DBoW2's L1Scoring::score (Thirdparty/DBoW2/DBoW2/ScoringObject.cpp:23-68)
 *                   bit for bit: the terms fabs(vi - wi) - fabs(vi) - fabs(wi) of the common words added in ascending word
 *                   order in double, then -score / 2.0 (an empty intersection gives -0.0). Every score is written,
 *                   including those of excluded keyframes.
 *   d_loop [B]      the selected database slot or -1; d_best [B] scoreBest.
 * Selection as the reference: scoreBest starts at 0.0; a keyframe that |d_db_id[n] - d_q_id[b]| < min_id_offset does not
 * exclude replaces the best only on score > scoreBest, so scores <= 0 never win and the first of equal scores does; a loop
 * is detected when a best exists and scoreBest > min_score. d_q_id / d_db_id are read only when min_id_offset > 0.
 * Two launches whatever B and N are; no allocation and no host synchronisation, so a CUDA graph may capture it. Checked
 * on the host: B, N, cap_q, cap_db < 0, NULL params or a NULL required pointer is SE2GPU_ERR_INVALID; cap_q above the
 * query's shared memory (12 bytes per word: 19 370 words on an H100) or N > 1 048 560 is SE2GPU_ERR_CAPACITY; a refused call writes
 * nothing. B == 0 does nothing. Like every device entry, it trusts the contents of device memory: counts within [0, cap]
 * (clamped) and ascending, unrepeated word ids. */
int se2gpu_detect_loop_device(int B, const int* d_q_word, const double* d_q_value, const int* d_q_n, int cap_q, int N,
                              const int* d_db_word, const double* d_db_value, const int* d_db_n, int cap_db, const int* d_q_id,
                              const int* d_db_id, const se2gpu_loop_detect_params* params, double* d_scores, int* d_loop,
                              double* d_best, void* stream);

/* VerifyLoopClose's verdict. GlobalMapper (localizer = 0) accepts when nMP >= min_match_mp && nGood >= min_match_kp &&
 * nMP * 1.0 / numMPsCurrent >= ratio_min_match_mp (GM_VCL_*, src/Config.cpp:76-78); the Localizer (localizer = 1) when
 * nGood >= min_match_kp (numMinMatch = 45). */
typedef struct se2gpu_loop_verify_params {
    int localizer;
    int min_match_mp;
    int min_match_kp;
    double ratio_min_match_mp;
} se2gpu_loop_verify_params;
#define SE2GPU_LOOP_VERIFY_GLOBAL_MAPPER {0, 15, 30, 0.05}
#define SE2GPU_LOOP_VERIFY_LOCALIZER {1, 0, 45, 0.0}

/* GlobalMapper::VerifyLoopClose (src/GlobalMapper.cpp:256-326) and Localizer::VerifyLoopClose (src/Localizer.cpp:394-431)
 * for B pairs, on DEVICE buffers, asynchronous on `stream`: pair b is keyframe b of `cur` against keyframe d_loop[b] of
 * `map` (d_loop as se2gpu_detect_loop_device writes it; -1 gives an empty pair, which is never verified).
 *   1. d_raw + b*cur->cap   SearchByBoW(cur, loop, mapMatch, false) with ORBmatcher()'s nnratio 0.6 and orientation check
 *                           (se2gpu_search_by_bow_batch_device on m, mp_only = 0), -1 = none.
 *   2. d_good + b*cur->cap  RemoveMatchOutlierRansac (:1207-1248): fewer than 10 raw matches clear everything; otherwise
 *                           cv::findFundamentalMat(FM_RANSAC, 3, 0.99) on keyPointsUn in ascending current-index order
 *                           (LMedS below 15, as OpenCV), the matches its mask keeps (none when it finds no model).
 *   3. d_mp + b*cur->cap    GlobalMapper only: RemoveKPMatch (:1251-1276) keeps a good match when
 *                           cur->has_mp[i] && map->has_mp[match]; all -1 for the Localizer, which does not call it.
 *                           In this entry has_mp is read as KeyFrame::hasObservation(idx) (mDualObservations), not
 *                           SearchByBoW's "map point non-null": step 1 runs with mp_only = 0 and never reads it.
 *   d_counts [B*3] (raw, good, MP) and d_verified [B] (1 = accepted, one byte per pair). d_n_mps_cur [B] is numMPsCurrent
 *   (getAllObsMPs().size()); it is read, like has_mp, only for the GlobalMapper verdict.
 * Launches: SearchByBoW's, one device-to-device copy, the outlier kernel and the verdict kernel, the same whatever B is; no
 * allocation and no host synchronisation. Checked on the host before anything is written:
 * B > the matcher's max_batch, cur->cap > max_queries or 8192 (the outlier kernel), map->cap > max_db is
 * SE2GPU_ERR_CAPACITY; a NULL handle, side, params or required pointer, or negative sizes, is SE2GPU_ERR_INVALID. B == 0
 * does nothing. Calls on one matcher are ordered like its other device entries. */
int se2gpu_verify_loop_device(se2gpu_matcher* m, int B, const se2gpu_bow_batch_kf* cur, const se2gpu_bow_batch_kf* map,
                              const int* d_loop, const int* d_n_mps_cur, const se2gpu_loop_verify_params* params, int* d_raw,
                              int* d_good, int* d_mp, int* d_counts, uint8_t* d_verified, void* stream);

/* ------------------------------------------------------------------------------------------ tracking */
/* Track::mTrack (reference src/Track.cpp:124-160) for up to max_streams independent camera streams, with the tracking state
 * (reference frame, mPrevMatched, mMatchIdx, mLocalMPs, mvbGoodPrl / mnGoodPrl, preSE2) kept on the device between calls
 * (DESIGN.md section 14). One se2gpu_tracker_step takes one frame per stream and runs, per stream and in the reference's
 * order, the extraction with the undistortion folded in, MatchByWindow(mRefFrame, mFrame, mPrevMatched, 20, mMatchIdx)
 * with nnratio 0.9, removeOutliers, updateFramePose with the pre-integration, doTriangulate (gated by nMinFrames) and
 * needNewKF. A stream without a reference frame runs mCreateFrame instead. updateFramePose, the pre-integration and
 * needNewKF run on the host in float / double as the reference does (glibc cosf / sinf); the device work of a step is
 * one CUDA graph, captured on the first step of each (B, w, h) and replayed after that. Keyframe creation, the local
 * mapper and covisibility stay with the caller. One handle per calling thread; calls on one handle are not re-entrant. */
typedef struct se2gpu_tracker se2gpu_tracker;

typedef struct se2gpu_tracker_params {
    int nfeatures;               /* Config::MaxFtrNumber: the extractor's nfeatures and needNewKF's c4 */
    float scale_factor;          /* Config::ScaleFactor */
    int nlevels;                 /* Config::MaxLevel */
    int fast_th;                 /* the extractor's FAST threshold (the reference's default is 20) */
    float K[9];                  /* Config::Kcam, row-major */
    float dist[12];              /* Config::Dcam; frames are raw, the undistortion is folded into extraction */
    int ndist;                   /* 0, 4, 5, 8 or 12 */
    se2gpu_grid_params grid;     /* Frame's grid bounds (static members, the same for every frame) */
    float lower_depth, upper_depth; /* Config::LOWER_DEPTH / UPPER_DEPTH */
    float cTb[16], bTc[16];      /* Config::cTb / bTc, row-major */
    float odo_noise[3];          /* Config::ODO_X_NOISE, ODO_Y_NOISE, ODO_T_NOISE */
    int min_frames;              /* nMinFrames (the reference: 8) */
    int max_frames;              /* nMaxFrames = Config::FPS */
} se2gpu_tracker_params;

/* the keyframe side of one stream for one step, from the caller's mpKF (read only for streams that track) */
typedef struct se2gpu_track_kf {
    const uint8_t* d_observed;   /* [nfeatures] mpKF->hasObservation(i), DEVICE (a slice of se2gpu_mp_keyframes fits) */
    const float* d_view_mp;      /* [nfeatures*3] mpKF->mViewMPs, DEVICE */
    int n_obs_mp;                /* mpKF->getSizeObsMP() */
    int accept_new_kf;           /* mpLocalMapper->acceptNewKF() */
    float odom[3];               /* mpKF->odom (x, y, theta) */
} se2gpu_track_kf;

/* what one step reports for one stream */
typedef struct se2gpu_track_result {
    int frame_id;                /* mFrame.id */
    int first;                   /* 1: the frame went through mCreateFrame */
    int n_keypoints;             /* mFrame.N */
    int n_matched;               /* MatchByWindow's count */
    int n_inlier;                /* removeOutliers' count, the nMatched needNewKF sees */
    int n_tracked_old;           /* doTriangulate's return (0 when gated) */
    int n_good_prl;              /* mnGoodPrl after the step (kept when gated) */
    int triangulated;            /* 1: doTriangulate passed the nMinFrames test */
    int new_kf;                  /* needNewKF() returned true, or a first frame has > 100 keypoints: the caller makes the
                                    keyframe, then calls se2gpu_tracker_reset */
    int abort_ba;                /* needNewKF called mpLocalMapper->setAbortBA() */
} se2gpu_track_result;

/* one stream's state: device arrays of nfeatures entries (the reference frame's and the current frame's keypoints and
 * descriptors, their counts, mPrevMatched [2 per entry], mMatchIdx, mLocalMPs [3 per entry], mvbGoodPrl) and host copies of
 * mFrame.Tcr, preSE2 (meas, cov column-major as Eigen stores it) and the ids */
typedef struct se2gpu_track_state {
    const se2gpu_keypoint* d_ref_kp; const uint8_t* d_ref_desc; const int* d_ref_n;
    const se2gpu_keypoint* d_cur_kp; const uint8_t* d_cur_desc; const int* d_cur_n;
    const float* d_prev; const int* d_matches; const float* d_local_mps; const uint8_t* d_good_prl;
    float Tcr[16];
    double pre_meas[3], pre_cov[9];
    int frame_id, kf_id, has_ref, n_good_prl;
} se2gpu_track_state;

/* max_w x max_h frames, up to max_streams (<= 65535) per step, on `device`. NULL on failure (se2gpu_last_error). */
se2gpu_tracker* se2gpu_tracker_create(int max_streams, int max_w, int max_h, const se2gpu_tracker_params* params, int device);
void se2gpu_tracker_destroy(se2gpu_tracker* t);
/* One step for streams 0 .. B-1 (the others are untouched): frames are 8-bit gray w x hgt, row stride `stride`, frame b at
 * frames + b*frame_stride, in DEVICE memory when frames_on_device != 0 and HOST memory otherwise; odom [B*3] (x, y, theta);
 * kf [B] the keyframe side (may be NULL when no stream 0 .. B-1 has a reference frame); out [B]. Synchronous: returns when
 * out is filled. Invalid input (B outside 1 .. max_streams, frames larger than the capacity, NULL pointers, a tracking
 * stream without its keyframe arrays) returns SE2GPU_ERR_INVALID / SE2GPU_ERR_CAPACITY and changes nothing. */
int se2gpu_tracker_step(se2gpu_tracker* t, int B, const uint8_t* frames, int frames_on_device, int w, int hgt, int stride,
                        size_t frame_stride, const float* odom, const se2gpu_track_kf* kf, se2gpu_track_result* out);
/* The same after dropping the reference frame of streams 0 .. B-1 and restarting their frame ids (Frame::nextId = 0): every
 * stream runs mCreateFrame. kf may be NULL. */
int se2gpu_tracker_first(se2gpu_tracker* t, int B, const uint8_t* frames, int frames_on_device, int w, int hgt, int stride,
                         size_t frame_stride, const float* odom, se2gpu_track_result* out);
/* resetLocalTrack (src/Track.cpp:191-204) for the n streams streams[0 .. n-1] (distinct), after the caller made their
 * current frame a keyframe: the reference frame becomes the current frame, mPrevMatched its keypoints, mLocalMPs
 * d_view_mp[j] [nfeatures*3] (DEVICE) up to its keypoint count and (-1,-1,-1) past it, mMatchIdx -1, preSE2 and mnGoodPrl
 * 0. A stream that has not extracted a frame since se2gpu_tracker_create, or a NULL pointer: SE2GPU_ERR_INVALID, nothing
 * changed. Asynchronous on the tracker's stream; the next call sees its results. */
int se2gpu_tracker_reset(se2gpu_tracker* t, int n, const int* streams, const float* const* d_view_mp);
/* stream b's state (device pointers stay valid for the life of the handle; read them after the call that wrote them) */
int se2gpu_tracker_state(se2gpu_tracker* t, int b, se2gpu_track_state* st);
/* nodes of the step graph last captured: kernels [1] and all nodes [1] (either may be NULL); 0 before the first step */
int se2gpu_tracker_graph_nodes(se2gpu_tracker* t, int* kernels, int* nodes);
/* test hook: eager != 0 runs every later step by direct launches on the tracker's stream instead of the captured graph */
int se2gpu_tracker_debug_eager(se2gpu_tracker* t, int eager);
/* Test hooks of the host part (no device needed), exactly what a step runs. _pose: updateFramePose's Tcr [16] and the
 * pre-integration of preSE2 (meas [3], cov [9] column-major, updated in place) for odometry odom / kf_odom / last_odom [3].
 * _decide: needNewKF's (bNeedNewKF && acceptNewKF, setAbortBA) for frame_id - kf_id = dframes. */
int se2gpu_track_host_pose(const se2gpu_tracker_params* p, const float* odom, const float* kf_odom, const float* last_odom,
                           float* Tcr, double* meas, double* cov);
int se2gpu_track_host_decide(const se2gpu_tracker_params* p, int dframes, int n_tracked_old, int n_obs_mp, int n_good_prl,
                             int n_inlier, const float* odom, const float* kf_odom, int accept_new_kf, int* new_kf, int* abort_ba);

/* ------------------------------------------------------------------------------------------ local BA */
typedef struct se2gpu_ba se2gpu_ba;

/* one entry per completed LM iteration (OptimizationAlgorithmLevenberg::solve call) */
typedef struct se2gpu_ba_iter_stats {
    double chi2_before; /* activeRobustChi2 at the start of the iteration */
    double chi2_after;  /* after the last accepted trial (== chi2_before if none) */
    double lambda;      /* damping after the iteration */
    double rho;         /* gain ratio of the last trial */
    int trials;         /* lambda trials used (1..10) */
    int accepted;       /* 1 if a trial was accepted */
    int terminate;      /* 1 if LM returned Terminate (10 failed trials or rho==0) */
    int pad;
} se2gpu_ba_iter_stats;

/* capacity-sized solver context on CUDA device `device` */
se2gpu_ba* se2gpu_ba_create(int max_poses, int max_points, int max_edges, int max_odo, int device);
void se2gpu_ba_destroy(se2gpu_ba* h);

/* Loads one local-BA window (what Map::loadLocalGraph + initializeOptimization(0) build):
 *   poses   [P*3]  VertexSE2 estimates (x,y,theta) of Twb; vertex id = index
 *   fixed   [P]    setFixed flags
 *   points  [L*3]  VertexSBAPointXYZ estimates (marginalised); landmarks without edges stay untouched
 *   edge_pose/edge_point [E], uv [E*2], info [E*3] (xx,xy,yy of the symmetric 2x2 information),
 *   odo_i/odo_j [O] PreEdgeSE2 vertices (error = Ri^T(rj-ri)-m), odo_meas [O*3], odo_info [O*6] (00,01,02,11,12,22)
 *   fx,cx,cy       CamPara (single focal length), Tcb [12] = row-major Rcb then tcb (SE3 of setExtParameter, inverted)
 *   huber_delta    RobustKernelHuber delta of every EdgeSE2XYZ
 * All HOST pointers; copies and re-indexes synchronously. A context may be loaded again with any window within its
 * capacities: a window with the loaded graph structure (vertices, fixed flags, edge endpoints, shard) only refreshes the
 * values, any other is rebuilt. On any error the context holds NO window: optimize, get, get_f32, reset and the debug
 * calls return SE2GPU_ERR_INVALID until a set_problem succeeds, and that one rebuilds. */
int se2gpu_ba_set_problem(se2gpu_ba* h, int P, int L, int E, int O, const double* poses, const uint8_t* fixed,
                          const double* points, const int* edge_pose, const int* edge_point, const double* uv,
                          const double* info, const int* odo_i, const int* odo_j, const double* odo_meas,
                          const double* odo_info, double fx, double cx, double cy, const double* Tcb,
                          double huber_delta);

/* optimize(max_iters): returns the number of LM iterations performed (like SparseOptimizer::optimize) or a
 * negative error. stop_flag (may be NULL) is polled between trials (setForceStopFlag). stats (may be NULL)
 * receives one entry per iteration. trace_poses [max_iters*P*3] / trace_points [max_iters*L*3] (may be NULL)
 * receive the estimates after each iteration (parity tests). */
int se2gpu_ba_optimize(se2gpu_ba* h, int max_iters, const volatile unsigned char* stop_flag,
                       se2gpu_ba_iter_stats* stats, double* trace_poses, double* trace_points);

/* The same for ONE g2o `solve(iteration)`-style slice of an optimisation: runs LM iterations first_iteration ..
 * first_iteration + max_iters - 1. lambda is initialised (1e-5 max|diag H|) at iteration 0 only; a call with first_iteration > 0
 * continues the lambda / nu schedule where the previous call on this context stopped, so optimize_from(0, 1), (1, 1), ... (9, 1)
 * is bit-identical to optimize(10). This is what a g2o::OptimizationAlgorithm subclass needs (INTEGRATION.md, option i). */
int se2gpu_ba_optimize_from(se2gpu_ba* h, int first_iteration, int max_iters, const volatile unsigned char* stop_flag,
                            se2gpu_ba_iter_stats* stats, double* trace_poses, double* trace_points);

/* Optimise B loaded windows together: window k is contexts[k] (distinct contexts, all on one device, world 1, a window
 * loaded, n <= 156 unknowns). Same semantics per window as se2gpu_ba_optimize(contexts[k], max_iters, ...): LM from
 * iteration 0, estimates and LM state left in the context, so get / get_f32 / reset work as after optimize.
 * stop_flags [B] (array and entries may be NULL) are polled between trials like setForceStopFlag. iterations [B]
 * receives each window's iteration count; stats [B * max_iters] (window k at k * max_iters), trace_poses [B] /
 * trace_points [B] (arrays of host pointers, may be NULL) as for se2gpu_ba_optimize. Ordered after the work already
 * enqueued on every context's stream; runs on contexts[0]'s stream and returns when all windows are done. Returns 0 or a
 * negative error; on a refusal no context changes, and the message names the offending window:
 *   SE2GPU_ERR_INVALID   a NULL or repeated context, contexts on different devices, a sharded context, no window loaded,
 *                        a context in multi-launch mode (se2gpu_ba_set_mode 1: the batch runs the persistent kernel);
 *   SE2GPU_ERR_CAPACITY  n > 156 unknowns (se2gpu_ba_optimize's band and envelope solvers take those), or max_iters above
 *                        a context's stats capacity.
 * Each window runs on one thread-block cluster of 8 CTAs (SE2GPU_BA_BATCH_CLUSTER: 2 or 4 for one context, for measuring),
 * one launch per cluster size present; a window's result equals se2gpu_ba_optimize's under SE2GPU_BA_PK_GRID = that size, byte for
 * byte, whatever it is batched with. Until the call returns, no other thread may use any of the contexts. */
int se2gpu_ba_optimize_batch(se2gpu_ba* const* contexts, int B, int max_iters,
                             const volatile unsigned char* const* stop_flags, int* iterations,
                             se2gpu_ba_iter_stats* stats, double* const* trace_poses, double* const* trace_points);
/* test hook: the cluster size the batched launch uses for the window loaded in h; changes nothing */
int se2gpu_ba_batch_cluster(se2gpu_ba* h);

/* restore the estimates loaded by the last se2gpu_ba_set_problem (device-side copy; lets a caller re-run
 * optimize on the same window without re-uploading it) */
int se2gpu_ba_reset(se2gpu_ba* h);

/* current estimates -> host (poses [P*3], points [L*3]) */
int se2gpu_ba_get(se2gpu_ba* h, double* poses, double* points);

/* Map::optimizeLocalGraph's write-back (reference src/Map.cpp:768-779) in the reference's storage type: poses [P*3] as
 * Se2(float x, float y, float theta) - theta narrowed to float, then normalised like Se2::Se2 (Config.cpp:194-195) - and
 * points [L*3] as cv::Point3f (toCvPt3f). Narrowed on the device; either pointer may be NULL. */
int se2gpu_ba_get_f32(se2gpu_ba* h, float* poses, float* points);

/* Map::loadLocalGraph's per-edge information matrix (reference src/Map.cpp:1024-1049), evaluated on the device from the
 * reference's own float data:
 *   Omega_e = (sigma_rot J_rotxy J_rotxy^T + sigma_z J_z J_z^T + mvLevelSigma2[octave_e] I)^-1,
 *   J_pi from view_mp[e] = pKF->mViewMPs[ftrIdx] and fx = Config::fxCam, Rcw = rows of pKF->Tcw(0:3,0:3),
 *   J_rotxy = (J_pi Rcw skew(lw - (Twb.x, Twb.y, 0)))[:, 0:2], J_z = -(J_pi Rcw)[:, 2],
 *   sigma_rot = 1/xrot_info, sigma_z = 1/z_info as float (Config::PLANEMOTION_XROT_INFO / _Z_INFO).
 * kf_Rcw [P*9], kf_twb_xy [P*2], mp_pos [L*3], view_mp [E*3], octave [E], level_sigma2 [nlevels]; info [E*3] receives
 * (xx, xy, yy) in double - the `info` argument of se2gpu_ba_set_problem. HOST pointers. */
int se2gpu_ba_build_information(int P, int L, int E, const float* view_mp, const int* edge_pose, const int* edge_point,
                                const int* octave, const float* kf_Rcw, const float* kf_twb_xy, const float* mp_pos,
                                const float* level_sigma2, int nlevels, float fx, float xrot_info, float z_info, double* info,
                                int device);

/* Multi-GPU: this context owns the landmarks j with j % world == rank (call before set_problem); the reduced
 * pose system [S | b | chi2 | scale] is summed over ranks once per LM trial through `allreduce`, which must
 * sum (op 0) or max (op 1) `count` doubles at device pointer `buf` in place across ranks, ordered on `stream`. */
typedef int (*se2gpu_allreduce_fn)(void* user, double* buf, size_t count, int op, void* stream);
int se2gpu_ba_set_shard(se2gpu_ba* h, int rank, int world, se2gpu_allreduce_fn allreduce, void* user);
/* Sharded runs on one NVLink node without any collective library on the data path: when the reduced system fits one CTA's
 * shared memory (<= 52 free poses) the whole optimize() of every rank is ONE persistent cooperative kernel, and the ranks'
 * kernels exchange through peer memory - twice per lambda-trial: the partial reduced systems [S | b] (every CTA of every rank
 * sums the ranks' buffers slice by slice over NVLink) and the scalars [chi2, scale, abort] - with flag words in peer memory
 * as the only synchronisation. The callback of se2gpu_ba_set_shard is then unused (it stays the path for larger windows).
 * One process per GPU: after se2gpu_ba_set_shard every rank calls _peer_export, the handles (SE2GPU_BA_PEER_HANDLE_BYTES
 * each, CUDA IPC) are all-gathered by the caller in rank order and passed to _peer_import. One process driving several
 * contexts (one per GPU, or several on one GPU for tests): _peer_attach_local on the array of contexts in rank order; every
 * context then needs its own host thread and stream, since the ranks' optimize() calls must run concurrently.
 * se2gpu_ba_optimize is a COLLECTIVE call in a sharded run (same arguments on every rank); stop_flag may differ per rank -
 * the abort decision is OR-ed over the ranks, so all of them stop after the same trial. A rank that does not show up within
 * SE2GPU_BA_PEER_TIMEOUT_S (default 10 s) makes the others return SE2GPU_ERR_CUDA instead of hanging. */
#define SE2GPU_BA_PEER_HANDLE_BYTES 128
int se2gpu_ba_peer_export(se2gpu_ba* h, void* handle_out);
int se2gpu_ba_peer_import(se2gpu_ba* h, const void* handles, int world);
int se2gpu_ba_peer_attach_local(se2gpu_ba** contexts, int world);
/* stream all BA work is enqueued on (cudaStream_t as void*); NULL = default stream */
int se2gpu_ba_set_stream(se2gpu_ba* h, void* stream);

/* parity/debug: linearise at the current estimate, Schur-reduce with damping `lambda`, solve; copy out whatever
 * is non-NULL. Hpp, S: [n*n] row-major (lower triangle valid), n = 3*#free poses; bp, bs, dx_p: [n];
 * Hll [L*9], bl [L*3], dx_l [L*3]; Hpl [E*9] (3x3 per edge, rows = pose, cols = point; original edge order).
 * Returns n (>=0) or a negative error. Does not change the estimates. */
/* execution mode of se2gpu_ba_optimize: 0 = auto (persistent cooperative kernel when available: single GPU, reduced system
 * fits one CTA's shared memory), 1 = one kernel per phase (always used for sharded runs), 2 = persistent or fail */
int se2gpu_ba_set_mode(se2gpu_ba* h, int mode);

/* per-kernel device timing for bench.py's roofline line; groups: 0 ba_linearize (+chi2 evaluation), 1 ba_pose_reduce,
 * 2 ba_lm_prep, 3 ba_schur, 4 ba_chol_solve, 5 ba_backsub_update, 6 ba_iter_begin/ba_decide, 7 ba_persistent (whole optimize),
 * 8 TMA staging of S inside the persistent kernel. In persistent mode groups 0-6 and 8 are in-kernel phase times of CTA 0. */
#define SE2GPU_BA_PROFILE_GROUPS 9
int se2gpu_ba_profile(se2gpu_ba* h, int enable);
int se2gpu_ba_profile_read(se2gpu_ba* h, double* ms, int* launches);

int se2gpu_ba_debug_system(se2gpu_ba* h, double lambda, double* chi2, double* Hpp, double* bp, double* Hll, double* bl,
                           double* Hpl, double* S, double* bs, double* dx_p, double* dx_l);

/* test hook: the host-side plan of the last set_problem that rebuilt the structure (a same-topology reload keeps it).
 * Writes min(n_out, SE2GPU_BA_PLAN_FIELDS) ints to `out` and returns SE2GPU_BA_PLAN_FIELDS; changes nothing.
 *   [0] nf (free poses)    [1] n = 3 nf
 *   [2] structure build: 0 dense nf x nf counting table, 1 comparison sort (nf * nf > 2^22)
 *   [3] envelope half-width w in pose blocks (max over block columns a of the last coupled block row - a)
 *   [4] reduced solve: 0 single-CTA shared-memory LDL^T, 1 two-CTA twisted solve (persistent kernel; one kernel per phase
 *       still uses 0), 2 partitioned band solver, 3 global-memory envelope factorisation
 *   [5] twisted split m0   [6] twisted separator width (0 when [4] != 1)
 *   [7] band half-width w  [8] band partition count p (0 when [4] != 2)
 *   [9] persistent grid (0 = no cooperative launch)   [10] Schur workers W of the persistent kernel
 *   [11] blocks of S       [12] most blocks one worker owns
 *   [13] workers whose blocks do not all fit the shared-memory cache (more than 16 blocks, or pair and edge lists beyond the
 *        arena): they run the sequential Schur sweep over lists in global memory */
#define SE2GPU_BA_PLAN_FIELDS 14
int se2gpu_ba_debug_plan(se2gpu_ba* h, int* out, int n_out);

/* se2gpu_ba_set_problem with every array in DEVICE memory (same arguments, same layout; Tcb stays a host pointer): the
 * graph structure (landmark sort, pose lists, block and pair lists of the reduced system, envelope) is built on the
 * device, and only O(free poses + blocks) ints come back for the host's solver decisions. The inputs are read on the
 * context's stream (se2gpu_ba_set_stream); the call returns once the window is loaded and the stream is synchronised, so
 * the caller may then overwrite them. Same contract as se2gpu_ba_set_problem: same-structure windows refresh the values
 * only, sharded contexts keep their landmarks, out-of-range endpoints return SE2GPU_ERR_INVALID (detected on the device),
 * capacity errors SE2GPU_ERR_CAPACITY, and on any error the context holds no window. The context ends up holding the
 * same device arrays, element for element, as after se2gpu_ba_set_problem of the same window. Loads by the other entry
 * point always rebuild the structure. */
int se2gpu_ba_set_problem_device(se2gpu_ba* h, int P, int L, int E, int O, const double* d_poses, const uint8_t* d_fixed,
                                 const double* d_points, const int* d_edge_pose, const int* d_edge_point, const double* d_uv,
                                 const double* d_info, const int* d_odo_i, const int* d_odo_j, const double* d_odo_meas,
                                 const double* d_odo_info, double fx, double cx, double cy, const double* Tcb,
                                 double huber_delta);

/* se2gpu_ba_build_information on DEVICE buffers of the caller's current device, asynchronous on `stream`. An edge whose
 * pose or landmark index is out of range gets NaN information (the host entry rejects the call instead). */
int se2gpu_ba_build_information_device(int P, int L, int E, const float* d_view_mp, const int* d_edge_pose,
                                       const int* d_edge_point, const int* d_octave, const float* d_kf_Rcw,
                                       const float* d_kf_twb_xy, const float* d_mp_pos, const float* d_level_sigma2,
                                       int nlevels, float fx, float xrot_info, float z_info, double* d_info, void* stream);

/* test hook: copies min(n_out, length) elements of one structure array the context holds on the device to `out` and
 * returns the array's length (for the double arrays: their raw 32-bit words, two per double), or SE2GPU_ERR_INVALID with
 * no window loaded. Changes nothing; the same after either load path. */
enum {
    SE2GPU_BA_STRUCT_HIDX, SE2GPU_BA_STRUCT_LM_PTR, SE2GPU_BA_STRUCT_PERM, SE2GPU_BA_STRUCT_E_POSE, SE2GPU_BA_STRUCT_E_HIDX,
    SE2GPU_BA_STRUCT_POSE_PTR, SE2GPU_BA_STRUCT_POSE_EDGES, SE2GPU_BA_STRUCT_POSE_ODO_PTR, SE2GPU_BA_STRUCT_POSE_ODO,
    SE2GPU_BA_STRUCT_BLK_A, SE2GPU_BA_STRUCT_BLK_B, SE2GPU_BA_STRUCT_BLK_PAIR_PTR, SE2GPU_BA_STRUCT_PAIR_E1,
    SE2GPU_BA_STRUCT_PAIR_E2, SE2GPU_BA_STRUCT_BLK_ODO_PTR, SE2GPU_BA_STRUCT_BLK_ODO, SE2GPU_BA_STRUCT_COLMAX,
    SE2GPU_BA_STRUCT_TW_CMAX1, SE2GPU_BA_STRUCT_BLK_ORDER, SE2GPU_BA_STRUCT_ENV_IDX, SE2GPU_BA_STRUCT_ODO_I,
    SE2GPU_BA_STRUCT_ODO_J, SE2GPU_BA_STRUCT_E_U, SE2GPU_BA_STRUCT_E_V, SE2GPU_BA_STRUCT_E_W00, SE2GPU_BA_STRUCT_E_W01,
    SE2GPU_BA_STRUCT_E_W11, SE2GPU_BA_STRUCT_ODO_M, SE2GPU_BA_STRUCT_ODO_W, SE2GPU_BA_STRUCT_COUNT
};
int se2gpu_ba_debug_structure(se2gpu_ba* h, int which, int* out, int n_out);

/* ------------------------------------------------------------------------------------------ pose-only BA */
/* Localizer::DoLocalBA (src/Localizer.cpp:233-302) for B independent problems, one CTA each, every LM iteration on the
 * device: one VertexSE3Expmap (estimate toSE3Quat(Tcw)), the plane-motion EdgeSE3ExpmapPrior of addPlaneMotionSE3Expmap
 * (src/optimizer.cpp:236-314) and one EdgeProjectXYZ2UV per edge (error uv - cam_map(T.map(xyz)), information info[e] * I,
 * RobustKernelHuber(huber_delta)), then g2o's optimize(iterations) with OptimizationAlgorithmLevenberg, in double precision
 * (DESIGN.md section 9). */
typedef struct se2gpu_pose_ba_params {
    float fx, cx, cy;       /* CamPara: Config::Kcam (0,0), (0,2), (1,2) */
    float Tbc[16];          /* Config::bTc, row-major 4x4 */
    float huber_delta;      /* Config::TH_HUBER */
    float xrot_info, yrot_info, z_info; /* Config::PLANEMOTION_XROT_INFO, _YROT_INFO, _Z_INFO (1e6, 1e6, 1) */
    int iterations;         /* optimize(iterations): 30 in DoLocalBA */
} se2gpu_pose_ba_params;

/* per-problem status */
#define SE2GPU_POSE_BA_OK 0
#define SE2GPU_POSE_BA_NO_EDGES 1  /* no projection edge: Tcw left as it is, 0 iterations */
#define SE2GPU_POSE_BA_NOT_PD 2    /* LM terminated because all 10 trials of its last iteration failed the Cholesky */
#define SE2GPU_POSE_BA_GATED 3     /* se2gpu_localizer_ba_device: no more edges than min_edges, Tcw left as it is */

/* HOST buffers, synchronous. Problem b owns edges edge_ptr[b] .. edge_ptr[b+1]-1 (edge_ptr [B+1], edge_ptr[0] = 0) of
 * xyz [E*3] (MapPoint::getPos), uv [E*2] (keyPointsUn[idx].pt) and info [E] (the scalar of the edge's information w*I).
 * Tcw [B*16] float row-major: in, the start estimate; out, toCvMat of the result (left as it is for NO_EDGES).
 * Optional (may be NULL): stats [B*iterations] (row b*iterations + k is iteration k; rows past iterations[b] are zero),
 * iterations [B] LM iterations done, status [B], pose [B*7] the double estimate (qx, qy, qz, qw, tx, ty, tz).
 * Device buffers are a per-device workspace that only grows. */
int se2gpu_pose_ba(int B, float* Tcw, const int* edge_ptr, const float* xyz, const float* uv, const float* info,
                   const se2gpu_pose_ba_params* params, se2gpu_ba_iter_stats* stats, int* iterations, int* status, double* pose,
                   int device);
/* The same on DEVICE buffers, asynchronous on `stream` (params is a host pointer, read during the call). d_stats rows past
 * an iteration count are not written. */
int se2gpu_pose_ba_device(int B, float* d_Tcw, const int* d_edge_ptr, const float* d_xyz, const float* d_uv, const float* d_info,
                          const se2gpu_pose_ba_params* params, se2gpu_ba_iter_stats* d_stats, int* d_iterations, int* d_status,
                          double* d_pose, void* stream);
/* parity hook: se2gpu_pose_ba plus trace [B*iterations*7], the estimate after every iteration (rows past the count zero) */
int se2gpu_pose_ba_debug_trace(int B, float* Tcw, const int* edge_ptr, const float* xyz, const float* uv, const float* info,
                               const se2gpu_pose_ba_params* params, se2gpu_ba_iter_stats* stats, int* iterations, int* status,
                               double* pose, double* trace, int device);

/* Localizer context: the device workspace for up to max_map_points local map points. One per calling thread. */
typedef struct se2gpu_localizer se2gpu_localizer;
se2gpu_localizer* se2gpu_localizer_create(int max_map_points, int device);
void se2gpu_localizer_destroy(se2gpu_localizer* h);
/* MatchLocalMap's observations + DoLocalBA on DEVICE buffers, asynchronous on `stream`, fed straight from
 * se2gpu_match_by_projection_device: d_kf_kp [n_kf] (*d_n_kf of them valid when d_n_kf is not NULL), d_matches_idx_mp [n_kf]
 * (-1 = unmatched), d_mp_xyz [n_mp*3] (getPos), d_mp_use [n_mp] (!isNull && isGoodPrl), d_inv_sigma2 [nlevels]
 * (mvInvLevelSigma2). The edges are the map points j with d_mp_use[j] that some keypoint matched, in ascending j; uv is
 * the keypoint of the highest index that matched j (repeated KeyFrame::addObservation keeps the last); every edge's
 * information is d_inv_sigma2[d_kf_kp[0].octave], which is what MapPoint::getOctave returns for the Localizer's new
 * keyframe (see DESIGN.md section 9). d_n_edges (may be NULL) receives the edge count; the optimisation runs only when it
 * exceeds min_edges (DoLocalBA's caller runs it above 30 observations), otherwise the status is GATED. d_Tcw [16] is
 * updated in place. d_stats [iterations], d_iterations, d_status [1], d_pose [7] may be NULL. */
int se2gpu_localizer_ba_device(se2gpu_localizer* h, const se2gpu_keypoint* d_kf_kp, int n_kf, const int* d_n_kf,
                               const int* d_matches_idx_mp, int n_mp, const float* d_mp_xyz, const uint8_t* d_mp_use,
                               const float* d_inv_sigma2, int nlevels, float* d_Tcw, const se2gpu_pose_ba_params* params,
                               int min_edges, int* d_n_edges, se2gpu_ba_iter_stats* d_stats, int* d_iterations, int* d_status,
                               double* d_pose, void* stream);

/* ------------------------------------------------------------------------------------------ localization */
/* Localizer::run (reference src/Localizer.cpp:32-176) for up to max_streams camera streams against one static map kept on
 * the device (DESIGN.md section 15). The map (keyframes, map points, observations, covisibility) goes up once at create;
 * the Localizer never edits it. One se2gpu_loc_step takes one frame and one odometry reading per stream and runs, per
 * stream: ReadFrameInfo (extraction, a new keyframe with no observations), UpdatePoseCurr on the host, and for a tracked
 * stream MatchLocalMap, DoLocalBA (above 30 observations), UpdateCovisKFCurr, UpdateLocalMap(1) and DetectIfLost. The
 * device work of a step is one CUDA graph per (B, w, h). Loop detection and verification stay with the caller, who runs
 * se2gpu_loc_relocalize for the streams it verified. The local map is in ascending map-point index. One handle per
 * calling thread; calls on one handle are not re-entrant.
 *
 * Not to be confused with se2gpu_localizer above, the pose-BA workspace. */
typedef struct se2gpu_loc se2gpu_loc;

/* the map, flattened (HOST arrays, copied once). K keyframes, M map points, keypoint slots in CSR. */
typedef struct se2gpu_loc_map {
    int n_kf, n_mp;
    const float* kf_Tcw;         /* [K*16] row-major keyframe poses */
    const int* kf_kp_ptr;        /* [K+1] keypoint slots of keyframe k: kf_kp_ptr[k] .. kf_kp_ptr[k+1]-1 */
    const int* kf_obs_mp;        /* [kf_kp_ptr[K]] map point of mDualObservations[idx], -1 for none */
    const int* kf_obs_ptr;       /* [K+1] CSR of mObservations: the map points keyframe k observes, strictly ascending */
    const int* kf_obs;
    const int* kf_cov_ptr;       /* [K+1] CSR of getAllCovisibleKFs() as keyframe indices, strictly ascending */
    const int* kf_cov;
    const float* mp_pos;         /* [M*3] getPos */
    const uint8_t* mp_null;      /* [M] isNull */
    const uint8_t* mp_good_prl;  /* [M] isGoodPrl */
    const uint8_t* mp_desc;      /* [M*32] mMainDescriptor */
    const int* mp_octave;        /* [M] mMainOctave, < nlevels */
} se2gpu_loc_map;

typedef struct se2gpu_loc_params {
    int nfeatures;               /* Config::MaxFtrNumber */
    float scale_factor;          /* Config::ScaleFactor */
    int nlevels;                 /* Config::MaxLevel, at most 16 */
    int fast_th;                 /* the extractor's FAST threshold */
    float K[9];                  /* Config::Kcam, row-major */
    float dist[12];              /* Config::Dcam; frames are raw, the undistortion is folded into extraction */
    int ndist;                   /* 0, 4, 5, 8 or 12 */
    se2gpu_grid_params grid;     /* Frame's grid origin and inverse cell sizes */
    float min_x, max_x, min_y, max_y; /* Frame::minXUn, maxXUn, minYUn, maxYUn (inImgBound, inclusive) */
    float cTb[16], bTc[16];      /* Config::cTb / bTc, row-major */
    se2gpu_pose_ba_params ba;    /* DoLocalBA: fx, cx, cy, Tbc (= bTc), TH_HUBER, plane-motion information, 30 iterations */
    float inv_level_sigma2[16];  /* mvInvLevelSigma2 [nlevels] */
    int max_local_mps;           /* per-stream capacity of the local map-point list */
} se2gpu_loc_params;

/* what a step (or a relocalization) reports for one stream */
typedef struct se2gpu_loc_result {
    int tracked;                 /* mbIsTracked after the call */
    int first;                   /* 1: the stream's first frame (mpKFRef == NULL): nothing but the extraction ran */
    int n_keypoints;             /* mpKFCurr->N */
    int n_matched;               /* MatchLocalMap's count (0 when it did not run) */
    int n_obs_mp;                /* mpKFCurr->getSizeObsMP() */
    int ba_status;               /* SE2GPU_POSE_BA_*: GATED at 30 observations or fewer, NO_EDGES when no BA ran */
    int ba_iterations;
    int n_local_kfs;             /* |mspKFLocal| */
    int n_local_mps;             /* |mspMPLocal|, the full count even when it exceeds max_local_mps */
    int overflow;                /* 1: n_local_mps > max_local_mps; every later call on this stream returns CAPACITY */
    float Tcw[16];               /* mpKFCurr->Tcw after the call, row-major (WriteTrajFile's source) */
} se2gpu_loc_result;

/* one stream's state: device arrays (current keypoints / descriptors [nfeatures] and their count, obs_mp [nfeatures] the
 * map point of each keypoint slot or -1, the local map-point list [max_local_mps] and its count, the local-keyframe
 * bitmap [K] and the covisible-keyframe bitmap [K] of the current keyframe) and host copies of Tcw and the flags */
typedef struct se2gpu_loc_stream_state {
    const se2gpu_keypoint* d_kp; const uint8_t* d_desc; const int* d_n;
    const int* d_obs_mp;
    const int* d_local_mps; const int* d_n_local_mps;
    const uint8_t* d_local_kfs; const uint8_t* d_covis_kfs;
    float Tcw[16];
    int has_frame, tracked, overflow;
} se2gpu_loc_stream_state;

/* Validates the map on the host before any allocation (indices in range, CSR monotone, octaves below nlevels): on any
 * failure SE2GPU_ERR_INVALID and NULL. max_streams <= 65535. */
se2gpu_loc* se2gpu_loc_create(int max_streams, int max_w, int max_h, const se2gpu_loc_params* params, const se2gpu_loc_map* map,
                              int device);
void se2gpu_loc_destroy(se2gpu_loc* h);
/* One frame for streams 0 .. B-1: frames as se2gpu_tracker_step, odom [B*3] (x, y, theta), out [B]. Synchronous. Invalid
 * input returns SE2GPU_ERR_INVALID / SE2GPU_ERR_CAPACITY and changes nothing; so does a step over a stream whose local
 * map overflowed (SE2GPU_ERR_CAPACITY). */
int se2gpu_loc_step(se2gpu_loc* h, int B, const uint8_t* frames, int frames_on_device, int w, int hgt, int stride,
                    size_t frame_stride, const float* odom, se2gpu_loc_result* out);
/* The verified branch of Localizer::run (Localizer.cpp:121-140) for the n distinct streams streams[j] whose last step
 * began lost (ran the else branch, where DetectLoopClose runs; a stream that lost tracking during its last step waits a
 * frame, as in the reference): setPose(kf_loop[j].Tcw), covisible = {kf_loop[j]}, UpdateLocalMap(3), MatchLoopClose over the pairs
 * match_curr / match_loop [match_ptr[j] .. match_ptr[j+1]) (idxCurr strictly ascending), DoLocalBA, MatchLocalMap,
 * DoLocalBA, DetectIfLost. out [n]; Tcw_first [n*16] (may be NULL) receives the pose after the first BA. Runs eagerly.
 * Bad input: SE2GPU_ERR_INVALID, nothing changed. A local map past max_local_mps marks the stream (out[j].overflow) and
 * returns SE2GPU_ERR_CAPACITY. */
int se2gpu_loc_relocalize(se2gpu_loc* h, int n, const int* streams, const int* kf_loop, const int* match_ptr, const int* match_curr,
                          const int* match_loop, se2gpu_loc_result* out, float* Tcw_first);
int se2gpu_loc_state(se2gpu_loc* h, int b, se2gpu_loc_stream_state* st);
/* nodes of the step graph last captured: kernels [1] and all nodes [1] (either may be NULL) */
int se2gpu_loc_graph_nodes(se2gpu_loc* h, int* kernels, int* nodes);
/* test hook: eager != 0 runs later steps by direct launches instead of the captured graph */
int se2gpu_loc_debug_eager(se2gpu_loc* h, int eager);
/* Test hook of the host part (no device needed): UpdatePoseCurr's Tcw [16] = cTb * Se2(ref_odom - odom).toCvSE3() * bTc *
 * ref_Tcw, exactly what a step computes. */
int se2gpu_loc_host_pose(const se2gpu_loc_params* p, const float* odom, const float* ref_odom, const float* ref_Tcw, float* Tcw);

/* ------------------------------------------------------------------------------------------ feature-graph constraints */
/* GlobalMapper::CreateFeatEdge (src/GlobalMapper.cpp:737-843) for B keyframe pairs, one CTA each, everything on the device:
 * the two-keyframe BA of OptKFPair / OptKFPairMatch (two VertexSE3 with the plane-motion EdgeSE3Prior of
 * addVertexSE3PlaneMotion, one marginalised VertexPointXYZ per point with a Huber EdgeSE3PointXYZ to each keyframe, g2o's
 * Levenberg-Marquardt with a Schur complement onto the poses), the chi2 outlier cut of OptKFPairMatch, and
 * Sparsifier::DoMarginalizeSE3XYZ + InfoSE3 (src/sparsifier.cpp:59-274) with their forward-difference Jacobians, in double
 * precision (DESIGN.md section 10).
 * mode 0 is CreateFeatEdge(from, to, cnstr): keyframe 0 fixed, iterations[0] LM iterations, at least min_points[0] points.
 * mode 1 is CreateFeatEdge(from, to, mapMatch, cnstr): both keyframes free, iterations[1] iterations, then every point with
 * an edge of chi2 > chi2_cut is an outlier and leaves the marginalisation; at least min_points[1] matches (counted before
 * the cut, as the reference does). A match belongs in the input only when both of its map points exist. */
typedef struct se2gpu_feat_edge_params {
    float Tbc[16];          /* Config::bTc, row-major 4x4 */
    float xrot_info, yrot_info, z_info; /* Config::PLANEMOTION_XROT_INFO, _YROT_INFO, _Z_INFO */
    float huber_delta;      /* RobustKernelHuber::setDelta(5.99) */
    int iterations[2];      /* optimize(15) in OptKFPair, optimize(30) in OptKFPairMatch */
    float chi2_cut;         /* dThreshChi2 = 5.0 */
    int min_points[2];      /* numMinMPs = 10; mapMatch.size() < 3 */
} se2gpu_feat_edge_params;
/* the reference's values, with an identity Tbc to be replaced by Config::bTc */
#define SE2GPU_FEAT_EDGE_PARAMS_INIT \
    { {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}, 1e6f, 1e6f, 1.f, 5.99f, {15, 30}, 5.0f, {10, 3} }

/* per-pair status */
#define SE2GPU_FEAT_EDGE_OK 0
#define SE2GPU_FEAT_EDGE_TOO_FEW 1  /* fewer points than min_points[mode]: the pair's outputs are left as they are */
#define SE2GPU_FEAT_EDGE_NOT_PD 2   /* LM ended on an iteration whose 10 trials all failed the Cholesky; the constraint is
                                       computed from the last accepted estimate */

/* HOST buffers, synchronous. Pair b owns points point_ptr[b] .. point_ptr[b+1]-1 (point_ptr [B+1], point_ptr[0] = 0, P =
 * point_ptr[B]). Tcw0 / Tcw1 [B*16] float row-major: KeyFrame::getPose() of the two keyframes. Per point: xyz [P*3] float,
 * the start estimate (MapPoint::getPos; in mode 1 of the point seen in keyframe 0); z0 / z1 [P*3] float, mViewMPs[idx] in
 * keyframe 0 / 1; info0 / info1 [P*9] double, mViewMPsInfo[idx], exactly as se2gpu_xyz_info writes them.
 * Outputs: measure [B*16] float (toCvMat of KF0^-1 KF1) and info [B*36] float (toCvMat6f), the SE3Constraint; optional (may
 * be NULL): status [B], iterations [B], stats [B*iterations[mode]] (rows past iterations[b] are zero), outlier [P] bytes
 * (mode 1; zero in mode 0), poses [B*14] (vSe3KFs: qx, qy, qz, qw, tx, ty, tz per keyframe, camera-to-world), points [P*3]
 * (every point's estimate, outliers included). Returns SE2GPU_ERR_INVALID before any launch on malformed input. */
int se2gpu_feat_edge(int B, int mode, const float* Tcw0, const float* Tcw1, const int* point_ptr, const float* xyz,
                     const float* z0, const float* z1, const double* info0, const double* info1,
                     const se2gpu_feat_edge_params* params, float* measure, float* info, int* status, int* iterations,
                     se2gpu_ba_iter_stats* stats, uint8_t* outlier, double* poses, double* points, int device);
/* The same on DEVICE buffers, asynchronous on `stream` (params is a host pointer, read during the call). d_info0 / d_info1
 * take se2gpu_xyz_info_device's outputs as they are. d_points [P*3] and d_work [P*3] doubles are required: the kernel keeps
 * the point estimates and the trial step there. d_stats rows past an iteration count are not written. d_point_ptr is device
 * memory and is trusted: it must start at 0 and ascend, and every array must hold d_point_ptr[B] points; the rejection of
 * malformed input described above is the host entry's. */
int se2gpu_feat_edge_device(int B, int mode, const float* d_Tcw0, const float* d_Tcw1, const int* d_point_ptr, const float* d_xyz,
                            const float* d_z0, const float* d_z1, const double* d_info0, const double* d_info1,
                            const se2gpu_feat_edge_params* params, float* d_measure, float* d_info, int* d_status,
                            int* d_iterations, se2gpu_ba_iter_stats* d_stats, uint8_t* d_outlier, double* d_poses,
                            double* d_points, double* d_work, void* stream);
/* parity hook: se2gpu_feat_edge plus trace [B*iterations[mode]*24], both keyframes' estimates (rotation row-major, then
 * translation) after every iteration (rows past the count zero) */
int se2gpu_feat_edge_debug_trace(int B, int mode, const float* Tcw0, const float* Tcw1, const int* point_ptr, const float* xyz,
                                 const float* z0, const float* z1, const double* info0, const double* info1,
                                 const se2gpu_feat_edge_params* params, float* measure, float* info, int* status, int* iterations,
                                 se2gpu_ba_iter_stats* stats, uint8_t* outlier, double* poses, double* points, double* trace,
                                 int device);

/* ------------------------------------------------------------------------------------------ global pose graph */
/* GlobalMapper::GlobalBA (src/GlobalMapper.cpp:328-535): one VertexSE3 per keyframe (camera-to-world, start value
 * toIsometry3D(cvu::inv(Tcw))) with the plane-motion EdgeSE3Prior of addVertexSE3PlaneMotion, one EdgeSE3 per odometry or
 * feature constraint (e = toVectorMQT(Z^-1 Xfrom^-1 Xto), information in the same [trans, rot] order), optimised by
 * Levenberg-Marquardt over the free vertices with a sparse direct solve, in double precision (DESIGN.md section 11). */
typedef struct se2gpu_global_ba_params {
    float Tbc[16];          /* Config::bTc, row-major 4x4 */
    float xrot_info, yrot_info, z_info; /* Config::PLANEMOTION_XROT_INFO, _YROT_INFO, _Z_INFO */
    int iterations;         /* Config::GLOBAL_ITER */
} se2gpu_global_ba_params;
/* the reference's values, with an identity Tbc to be replaced by Config::bTc */
#define SE2GPU_GLOBAL_BA_PARAMS_INIT \
    { {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}, 1e6f, 1e6f, 1.f, 15 }

#define SE2GPU_GLOBAL_BA_OK 0
#define SE2GPU_GLOBAL_BA_NOT_PD 2  /* LM ended on an iteration whose 10 trials all met a pivot block that is not positive
                                      definite; the poses are the last accepted estimate */

/* A context: grow-only device buffers for the plan and the solver, a page-locked staging arena and a stream, on device
 * `device`. One context serves graphs of any size and topology; a call gives the same bytes as on a fresh context. Calls
 * on one context may use different streams: each call's work waits for the previous call's kernel on the device. */
typedef struct se2gpu_global_ba_ctx se2gpu_global_ba_ctx;
se2gpu_global_ba_ctx* se2gpu_global_ba_create(int device);
void se2gpu_global_ba_destroy(se2gpu_global_ba_ctx* h);

/* HOST buffers, synchronous. N keyframes: Tcw [N*16] float row-major (KeyFrame::Tcw), fixed [N] (mIdKF == 0). E edges:
 * edge_from / edge_to [E] vertex indices, measure [E*16] float (SE3Constraint::measure), info [E*36] float (its info).
 * Outputs: Tcw_out [N*16] float (the pose setPose receives: cvu::inv(toCvMat(estimate))); optional (may be NULL): status,
 * iterations, stats [params->iterations] (rows past the count are zero), poses [N*7] (the estimates as SE3Quat: qx, qy, qz,
 * qw, tx, ty, tz, camera-to-world). With no free vertex no iteration runs, as in g2o. Returns SE2GPU_ERR_INVALID before any
 * launch when N <= 0, an index is out of range, from == to, or a measurement or information is not finite or an
 * information is not symmetric. */
int se2gpu_global_ba(se2gpu_global_ba_ctx* h, int N, const float* Tcw, const uint8_t* fixed, int E, const int* edge_from,
                     const int* edge_to, const float* measure, const float* info, const se2gpu_global_ba_params* params,
                     float* Tcw_out, int* status, int* iterations, se2gpu_ba_iter_stats* stats, double* poses);
/* The same on DEVICE values, asynchronous on `stream`. The topology (fixed, edge_from, edge_to) is HOST memory: the
 * ordering and the gather lists are planned on the host once per call. d_edge_status [E] (may be NULL) leaves out every
 * edge whose entry is SE2GPU_FEAT_EDGE_TOO_FEW, so se2gpu_feat_edge_device can write the feature edges' d_measure / d_info /
 * d_status straight into slices of these arrays; such an edge keeps its place in the plan and contributes nothing. The
 * values are trusted: the finiteness and symmetry checks are the host entry's. */
int se2gpu_global_ba_device(se2gpu_global_ba_ctx* h, int N, const float* d_Tcw, const uint8_t* fixed, int E, const int* edge_from,
                            const int* edge_to, const float* d_measure, const float* d_info, const int* d_edge_status,
                            const se2gpu_global_ba_params* params, float* d_Tcw_out, int* d_status, int* d_iterations,
                            se2gpu_ba_iter_stats* d_stats, double* d_poses, void* stream);
/* Phase timing of the kernel (a measurement aid; it adds a %globaltimer read per phase on one thread). on = 1 zeroes and
 * starts it, on = 0 stops it. profile_read waits for the last call and returns ms [7], the time accumulated since
 * profiling started in: setup (start values, priors, first chi2), linearisation, gather of H and b, copy and damping,
 * factorisation, substitution, and trial (oplus, computeScale, chi2 at the trial state, the LM decision). */
int se2gpu_global_ba_profile(se2gpu_global_ba_ctx* h, int on);
int se2gpu_global_ba_profile_read(se2gpu_global_ba_ctx* h, double* ms);
/* GlobalBA's map-point write-back: pos_out [M*3] = Rwc * view_mp + twc of keyframe kf_index[m], Twc the rigid inverse of
 * Tcw [N*16] (normally se2gpu_global_ba's Tcw_out), in float. view_mp [M*3] is mViewMPs[idx] of the point's main keyframe.
 * HOST buffers, synchronous; kf_index is checked against N. */
int se2gpu_global_ba_update_points(int M, const int* kf_index, const float* view_mp, int N, const float* Tcw, float* pos_out,
                                   int device);
/* the same on DEVICE buffers, asynchronous on `stream`; d_kf_index is trusted */
int se2gpu_global_ba_update_points_device(int M, const int* d_kf_index, const float* d_view_mp, const float* d_Tcw, float* d_pos_out,
                                          void* stream);

/* ------------------------------------------------------------------------------------------ SE(3)-XYZ window BA */
/* The window of Map::loadLocalGraph (src/Map.cpp:414-566) and Map::loadLocalGraphOnlyBa (:568-698) under g2o's
 * Levenberg-Marquardt, as LocalMapper::removeOutlierChi2 (src/LocalMapper.cpp:172-230) and the TIME_TO_LOG_LOCAL_BA timing
 * (:251-276) run it, in double precision (DESIGN.md section 12). One VertexSE3Expmap per keyframe (estimate toSE3Quat(Tcw)),
 * with the plane-motion EdgeSE3ExpmapPrior of addPlaneMotionSE3Expmap where prior[k] is set; one EdgeSE3Expmap per odometry
 * link (vertices[0] = from, vertices[1] = to, e = log(T_to^-1 Z T_from), information permuted from [trans rot] to
 * [rot trans] as addEdgeSE3Expmap does); one marginalised VertexSBAPointXYZ per map point and one EdgeProjectXYZ2UV per
 * observation (information inv_sigma2 * I, RobustKernelHuber(huber_delta)). loadLocalGraphOnlyBa is the same call with
 * every prior[k] = 0 and no odometry. */
typedef struct se2gpu_se3_ba_params {
    float fx, cx, cy;       /* CamPara: Config::Kcam (0,0), (0,2), (1,2) */
    float Tbc[16];          /* Config::bTc, row-major 4x4 */
    float huber_delta;      /* Config::TH_HUBER */
    float xrot_info, yrot_info, z_info; /* Config::PLANEMOTION_XROT_INFO, _YROT_INFO, _Z_INFO */
    int iterations;         /* optimize(iterations): 10 in removeOutlierChi2, LOCAL_ITER in the timing path */
    float chi2_cut;         /* an edge is an outlier when its raw chi2 e^T Omega e exceeds this: 25 in removeOutlierChi2 */
} se2gpu_se3_ba_params;

#define SE2GPU_SE3_BA_OK 0
#define SE2GPU_SE3_BA_NOT_PD 2  /* LM ended on an iteration whose 10 trials all met a pivot block that is not positive
                                   definite; the estimates are the last accepted ones */

/* A context: grow-only device buffers for the plan and the solver, a page-locked staging arena and a stream, on device
 * `device`. One context serves windows of any size and topology; a call gives the same bytes as on a fresh context. Calls
 * on one context may use different streams: each call's work waits for the previous call's kernel on the device. */
typedef struct se2gpu_se3_ba_ctx se2gpu_se3_ba_ctx;
se2gpu_se3_ba_ctx* se2gpu_se3_ba_create(int device);
void se2gpu_se3_ba_destroy(se2gpu_se3_ba_ctx* h);

/* HOST buffers, synchronous. N keyframes: Tcw [N*16] float row-major, fixed [N] (nonzero: fixed vertex), prior [N] (nonzero:
 * the keyframe has the plane-motion prior). O odometry links: odo_from / odo_to [O], odo_measure [O*16] float
 * (mOdoMeasureFrom.second.measure), odo_info [O*36] float in KeyFrame's [trans rot] order. L points: xyz [L*3] float. E edges:
 * edge_point / edge_kf [E], uv [E*2] float (keyPointsUn[idx].pt), inv_sigma2 [E] (mvInvLevelSigma2[octave]).
 * Outputs: chi2 [E] the raw chi2 of every edge at the final estimate, outlier [E] (chi2 > params->chi2_cut). Optional (may
 * be NULL): status, iterations, stats [params->iterations] (rows past the count are zero), poses [N*7] (qx, qy, qz, qw, tx,
 * ty, tz), points [L*3] double, Tcw_out [N*16] float (toCvMat of the estimate), xyz_out [L*3] float. A fixed keyframe
 * and a keyframe no edge touches come back in Tcw_out bit for bit as they went in; a point without edges is not in the
 * optimised graph and comes back as it was. With no free vertex no iteration runs, as in g2o. Returns
 * SE2GPU_ERR_INVALID before any launch when N <= 0, a count is negative, an index is out of range, an odometry link has
 * from == to, a point has two edges to one keyframe, a value or parameter is not finite (chi2_cut may be infinite), an
 * odometry information is not symmetric or an inv_sigma2 is not positive. */
int se2gpu_se3_ba(se2gpu_se3_ba_ctx* h, int N, const float* Tcw, const uint8_t* fixed, const uint8_t* prior, int O, const int* odo_from,
                  const int* odo_to, const float* odo_measure, const float* odo_info, int L, const float* xyz, int E,
                  const int* edge_point, const int* edge_kf, const float* uv, const float* inv_sigma2,
                  const se2gpu_se3_ba_params* params, double* chi2, uint8_t* outlier, int* status, int* iterations,
                  se2gpu_ba_iter_stats* stats, double* poses, double* points, float* Tcw_out, float* xyz_out);
/* The same on DEVICE values and outputs, asynchronous on `stream` (every output may be NULL). The topology (fixed, prior,
 * odo_from, odo_to, edge_point, edge_kf) is HOST memory and is checked; the values are trusted. */
int se2gpu_se3_ba_device(se2gpu_se3_ba_ctx* h, int N, const float* d_Tcw, const uint8_t* fixed, const uint8_t* prior, int O,
                         const int* odo_from, const int* odo_to, const float* d_odo_measure, const float* d_odo_info, int L,
                         const float* d_xyz, int E, const int* edge_point, const int* edge_kf, const float* d_uv,
                         const float* d_inv_sigma2, const se2gpu_se3_ba_params* params, double* d_chi2, uint8_t* d_outlier,
                         int* d_status, int* d_iterations, se2gpu_ba_iter_stats* d_stats, double* d_poses, double* d_points,
                         float* d_Tcw_out, float* d_xyz_out, void* stream);
/* parity hook: se2gpu_se3_ba plus trace [iterations * (N*7 + L*3)], the estimate after every iteration (the N poses, then
 * the L points; rows past the count zero) */
int se2gpu_se3_ba_debug_trace(se2gpu_se3_ba_ctx* h, int N, const float* Tcw, const uint8_t* fixed, const uint8_t* prior, int O,
                              const int* odo_from, const int* odo_to, const float* odo_measure, const float* odo_info, int L,
                              const float* xyz, int E, const int* edge_point, const int* edge_kf, const float* uv,
                              const float* inv_sigma2, const se2gpu_se3_ba_params* params, double* chi2, uint8_t* outlier,
                              int* status, int* iterations, se2gpu_ba_iter_stats* stats, double* poses, double* points,
                              double* trace);

#ifdef __cplusplus
}
#endif
#endif /* SE2GPU_H */
