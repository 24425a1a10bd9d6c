"""Loop closure on the device: GlobalMapper / Localizer DetectLoopClose and VerifyLoopClose for a batch of query
keyframes (reference src/GlobalMapper.cpp:201-326, src/Localizer.cpp:337-431) over the C ABI.

`detect_loop_device` scores every query against every database keyframe with DBoW2's L1 metric and selects the loop
keyframe (se2gpu_detect_loop_device); `verify_loop_device` matches each query with its loop keyframe, rejects outliers with
the fundamental-matrix RANSAC and applies the acceptance test (se2gpu_verify_loop_device). Both take device pointers
(ints or torch tensors) in the layouts Vocabulary.compute_bow_device writes and run asynchronously on `stream`.
"""
from __future__ import annotations

import ctypes as C

from ._capi import LoopDetectParams, LoopVerifyParams, check, lib, ptr

# GM_DCL_MIN_KFID_OFFSET, GM_DCL_MIN_SCORE_BEST (src/Config.cpp:80-81); the Localizer's 0.05 with no keyframe excluded
DETECT_GLOBAL_MAPPER = (20, 0.005)
DETECT_LOCALIZER = (0, 0.05)
# (localizer, GM_VCL_NUM_MIN_MATCH_MP, GM_VCL_NUM_MIN_MATCH_KP or the Localizer's numMinMatch, GM_VCL_RATIO_MIN_MATCH_MP)
VERIFY_GLOBAL_MAPPER = (0, 15, 30, 0.05)
VERIFY_LOCALIZER = (1, 0, 45, 0.0)


def _stream(stream):
    return C.c_void_p(int(stream) if stream else 0)


def detect_loop_device(B, d_q_word, d_q_value, d_q_n, cap_q, N, d_db_word, d_db_value, d_db_n, cap_db, d_scores, d_loop, d_best,
                       d_q_id=None, d_db_id=None, params=DETECT_GLOBAL_MAPPER, stream=0):
    """DetectLoopClose for B queries against N database keyframes (slots in ascending keyframe id): d_scores [B*N] float64
    every L1 score, d_loop [B] int32 the selected slot or -1, d_best [B] float64 scoreBest. params = (min_id_offset,
    min_score); the ids are read only when min_id_offset > 0. See se2gpu_detect_loop_device."""
    p = LoopDetectParams(int(params[0]), float(params[1]))
    check(lib().se2gpu_detect_loop_device(int(B), ptr(d_q_word), ptr(d_q_value), ptr(d_q_n), int(cap_q), int(N), ptr(d_db_word),
                                          ptr(d_db_value), ptr(d_db_n), int(cap_db), ptr(d_q_id), ptr(d_db_id), C.byref(p),
                                          ptr(d_scores), ptr(d_loop), ptr(d_best), _stream(stream)), "se2gpu_detect_loop_device")


def verify_loop_device(matcher, B, cur, map_, d_loop, d_raw, d_good, d_mp, d_counts, d_verified, d_n_mps_cur=None,
                       params=VERIFY_GLOBAL_MAPPER, stream=0):
    """VerifyLoopClose for B pairs: query b of `cur` against slot d_loop[b] of `map_` (ORBmatcher.BowBatchSide structs; has_mp
    is hasObservation(idx), needed for the GlobalMapper verdict). d_raw / d_good / d_mp [B*cur.cap] int32 (-1 = none),
    d_counts [B*3] int32 (raw, good, MP), d_verified [B] uint8. `matcher` is an ORBmatcher with a batch context.
    See se2gpu_verify_loop_device."""
    assert matcher.h, "verify_loop_device needs an ORBmatcher with a context (pass max_queries / max_db / max_batch)"
    p = LoopVerifyParams(int(params[0]), int(params[1]), int(params[2]), float(params[3]))
    check(lib().se2gpu_verify_loop_device(matcher.h, int(B), C.byref(cur), C.byref(map_), ptr(d_loop), ptr(d_n_mps_cur), C.byref(p),
                                          ptr(d_raw), ptr(d_good), ptr(d_mp), ptr(d_counts), ptr(d_verified), _stream(stream)),
          "se2gpu_verify_loop_device")
