"""Status codes of the host-buffer entry points and of the handle-less _device entry points.

Every host-buffer entry selects its device through one staging helper, and every handle-less _device entry checks for
a device through one test, so the three outcomes must agree across modules: a machine without a GPU gives
SE2GPU_ERR_NO_DEVICE, a device index one past the last gives SE2GPU_ERR_INVALID (SE2GPU_ERR_NO_DEVICE without a GPU), and
a null or out-of-range argument gives SE2GPU_ERR_INVALID on either kind of machine. On a machine with a GPU the _device
entries only see invalid arguments, which are rejected before any launch: no kernel is handed a host pointer.
"""
import ctypes as C

import numpy as np
import pytest

from se2lam_b200 import _capi, build
from se2lam_b200._capi import KP_DTYPE, BA_STATS_DTYPE, PoseBAParams

OK, NO_DEVICE, CUDA, INVALID = 0, -1, -2, -3
N = 8


@pytest.fixture(scope="module")
def lib():
    build.build_lib()
    return _capi.lib()


@pytest.fixture(scope="module")
def has_gpu(lib):
    return lib.se2gpu_device_count() > 0


def p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def f32(*shape):
    return np.zeros(shape, np.float32)


def i32(*shape):
    return np.zeros(shape, np.int32)


def u8(*shape):
    return np.zeros(shape, np.uint8)


def kps(n):
    return np.zeros(n, KP_DTYPE)


def pose_params(iterations=2):
    prm = PoseBAParams()
    prm.fx, prm.cx, prm.cy, prm.huber_delta = 500.0, 320.0, 240.0, 5.991 ** 0.5
    for k in (0, 5, 10, 15):
        prm.Tbc[k] = 1.0
    prm.xrot_info = prm.yrot_info = prm.z_info = 1e6
    prm.iterations = iterations
    return prm


# host-buffer entries: name -> call(L, device, valid) with valid, non-empty arguments or one bad argument
def _triangulate(L, dev, valid):
    idx = i32(N) if valid else np.full(N, 2, np.int32)        # 2 projections: index 2 is out of range
    return L.se2gpu_triangulate(N, p(f32(2 * N)), p(f32(2 * N)), p(f32(2, 12)), 2, p(idx), p(i32(N)), p(f32(3 * N)), dev)


def _track_triangulate(L, dev, valid):
    return L.se2gpu_track_triangulate(p(kps(N)), N, p(kps(N)), N, p(i32(N)), p(u8(N)), p(f32(3 * N)), p(f32(16)), p(f32(9)),
                                      0.1, 10.0, 2 if valid else 0, p(f32(3 * N)), p(u8(N)), p(i32(2)), dev)


def _xyz_info(L, dev, valid):
    pose = i32(N) if valid else np.full(N, 1, np.int32)       # 1 pose: index 1 is out of range
    return L.se2gpu_xyz_info(N, p(f32(3 * N)), p(pose), p(i32(N)), p(f32(16)), 1, 500.0, p(np.zeros(9 * N)),
                             p(np.zeros(9 * N)), dev)


def _projection_observations(L, dev, valid):
    m = np.full(N, 0 if valid else 1, np.int32)               # 1 map point: index 1 is out of range
    return L.se2gpu_projection_observations(p(kps(N)), N, p(m), p(f32(16)), p(f32(2)), p(i32(1)), p(i32(1)), p(f32(3)),
                                            p(f32(1)), p(f32(1)), 1, p(f32(16)), 1, p(f32(9)), 0.1, 10.0, 500.0, p(u8(N)),
                                            p(f32(3 * N)), p(np.zeros(9 * N)), dev)


def _debug_svd4(L, dev, valid):
    return L.se2gpu_debug_svd4(N, p(f32(16 * N)) if valid else None, p(f32(4 * N)), p(f32(16 * N)), dev)


def _remove_outliers(L, dev, valid):
    m = np.full(N, -1 if valid else N, np.int32)              # N frame-2 keypoints: index N is out of range
    return L.se2gpu_remove_outliers(1, p(kps(N)), None, N, p(kps(N)), None, N, p(m), p(i32(1)), None, None, dev)


def _fundam_debug_niters(L, dev, valid):
    n = np.array([10 if valid else 0], np.int32)              # n must be positive
    return L.se2gpu_fundam_debug_niters(1, p(n), p(i32(1)), p(np.array([5], np.int32)), p(i32(1)), dev)


def _pose_ba(L, dev, valid, trace=False):
    edge_ptr = np.array([0, 2] if valid else [1, 2], np.int32)  # edge_ptr[0] must be 0
    prm = pose_params()
    args = [1, p(np.eye(4, dtype=np.float32)), p(edge_ptr), p(f32(2, 3)), p(f32(2, 2)), p(f32(2)), C.cast(C.pointer(prm), C.c_void_p),
            p(np.zeros(prm.iterations, BA_STATS_DTYPE)), p(i32(1)), p(i32(1)), p(np.zeros(7))]
    if trace:
        return L.se2gpu_pose_ba_debug_trace(*args, p(np.zeros(7 * prm.iterations)), dev)
    return L.se2gpu_pose_ba(*args, dev)


def _median_descriptor(L, dev, valid):
    ptr = np.array([0, 2] if valid else [2, 0], np.int32)     # ptr must be non-decreasing
    return L.se2gpu_median_descriptor(p(u8(2, 32)), p(ptr), 1, p(i32(1)), p(i32(1)), dev)


def _hamming_distance(L, dev, valid):
    return L.se2gpu_hamming_distance(p(u8(N, 32)) if valid else None, p(u8(N, 32)), N, p(i32(N)), dev)


def _orb_debug_nth(L, dev, valid):
    values = np.arange(4, dtype=np.uint32) if valid else None
    return L.se2gpu_orb_debug_nth_element(p(values), p(np.array([0, 4], np.int32)), p(np.array([1], np.int32)), 1, dev)


def _orb_debug_nth_f32(L, dev, valid):
    values = np.arange(4, dtype=np.float32) if valid else None
    return L.se2gpu_orb_debug_nth_element_f32(p(values), p(np.array([0, 4], np.int32)), p(np.array([1], np.int32)), 1, p(i32(4)), dev)


def _ba_build_information(L, dev, valid):
    point = np.array([0 if valid else 1], np.int32)           # 1 landmark: index 1 is out of range
    return L.se2gpu_ba_build_information(1, 1, 1, p(np.array([0, 0, 1], np.float32)), p(i32(1)), p(point), p(i32(1)),
                                         p(np.eye(3, dtype=np.float32)), p(f32(2)), p(f32(3)), p(np.ones(1, np.float32)), 1,
                                         500.0, 1e6, 1e6, p(np.zeros(3)), dev)


HOST_ENTRIES = {
    "triangulate": _triangulate,
    "track_triangulate": _track_triangulate,
    "xyz_info": _xyz_info,
    "projection_observations": _projection_observations,
    "debug_svd4": _debug_svd4,
    "remove_outliers": _remove_outliers,
    "fundam_debug_niters": _fundam_debug_niters,
    "pose_ba": _pose_ba,
    "pose_ba_debug_trace": lambda L, dev, valid: _pose_ba(L, dev, valid, trace=True),
    "median_descriptor": _median_descriptor,
    "hamming_distance": _hamming_distance,
    "orb_debug_nth_element": _orb_debug_nth,
    "orb_debug_nth_element_f32": _orb_debug_nth_f32,
    "ba_build_information": _ba_build_information,
}


@pytest.mark.parametrize("name", sorted(HOST_ENTRIES))
def test_host_entry_without_device(lib, has_gpu, name):
    if has_gpu:
        pytest.skip("GPU present")
    assert HOST_ENTRIES[name](lib, 0, True) == NO_DEVICE, _capi.last_error()


@pytest.mark.parametrize("name", sorted(HOST_ENTRIES))
def test_host_entry_device_past_the_last(lib, has_gpu, name):
    rc = HOST_ENTRIES[name](lib, lib.se2gpu_device_count(), True)
    assert rc == (INVALID if has_gpu else NO_DEVICE), _capi.last_error()


@pytest.mark.parametrize("name", sorted(HOST_ENTRIES))
def test_host_entry_bad_argument(lib, name):
    assert HOST_ENTRIES[name](lib, 0, False) == INVALID, _capi.last_error()


def test_voc_transform_null_vocabulary(lib):
    assert lib.se2gpu_voc_transform(None, p(u8(N, 32)), N, 4, p(i32(N)), p(np.zeros(N)), None) == INVALID


# handle-less _device entries: the pointers of a valid call are host memory, which only a machine without a GPU is handed
def _dev_triangulate(L, valid):
    a = [p(f32(16 * N)) if valid else None] * 6
    return L.se2gpu_triangulate_device(N, *a, None)


def _dev_track_triangulate(L, valid):
    return L.se2gpu_track_triangulate_device(p(kps(N)), N, None, p(kps(N)), p(i32(N)), p(u8(N)), p(f32(3 * N)), p(f32(16)),
                                             p(f32(9)), 0.1, 10.0, 2, p(f32(3 * N)), p(u8(N)), p(i32(2)) if valid else None, None)


def _dev_xyz_info(L, valid):
    a = p(f32(16 * N)) if valid else None
    return L.se2gpu_xyz_info_device(N, a, p(i32(N)), p(i32(N)), p(f32(16)), 500.0, p(np.zeros(9 * N)), p(np.zeros(9 * N)), None)


def _dev_projection_observations(L, valid):
    a = p(f32(16 * N)) if valid else None
    return L.se2gpu_projection_observations_device(p(kps(N)), N, None, p(i32(N)), *([a] * 9), 0.1, 10.0, 500.0, p(u8(N)),
                                                   p(f32(3 * N)), p(np.zeros(9 * N)), None)


def _dev_remove_outliers(L, valid):
    return L.se2gpu_remove_outliers_device(1, p(kps(N)), None, N, p(kps(N)), None, N, p(i32(N)), p(i32(1)) if valid else None,
                                           None, None, None)


def _dev_pose_ba(L, valid):
    prm = pose_params()
    return L.se2gpu_pose_ba_device(1, p(np.eye(4, dtype=np.float32)) if valid else None, p(np.array([0, 2], np.int32)),
                                   p(f32(2, 3)), p(f32(2, 2)), p(f32(2)), C.cast(C.pointer(prm), C.c_void_p), None, None, None,
                                   None, None)


def _dev_keypoints_to_points(L, valid):
    return L.se2gpu_keypoints_to_points_device(p(kps(N)), N, None, p(f32(2 * N)) if valid else None, None)


DEVICE_ENTRIES = {
    "triangulate_device": _dev_triangulate,
    "track_triangulate_device": _dev_track_triangulate,
    "xyz_info_device": _dev_xyz_info,
    "projection_observations_device": _dev_projection_observations,
    "remove_outliers_device": _dev_remove_outliers,
    "pose_ba_device": _dev_pose_ba,
    "keypoints_to_points_device": _dev_keypoints_to_points,
}


@pytest.mark.parametrize("name", sorted(DEVICE_ENTRIES))
def test_device_entry_without_device(lib, has_gpu, name):
    if has_gpu:
        pytest.skip("GPU present")
    assert DEVICE_ENTRIES[name](lib, True) == NO_DEVICE, _capi.last_error()


@pytest.mark.parametrize("name", sorted(DEVICE_ENTRIES))
def test_device_entry_bad_argument(lib, name):
    assert DEVICE_ENTRIES[name](lib, False) == INVALID, _capi.last_error()
