"""The CameraCalibration::rectifyImage drop-in (ov2slam_b200/host/camera_calibration_rect_gpu.cpp): its host-side flow with the
device call mocked (CPU), its compile check against the reference's own headers, and its self-test on the device against
cv2.remap (GPU)."""
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import remap_ref as RR
from ov2slam_b200 import build

ROOT = Path(__file__).resolve().parents[1]


def _write_input(path, img, m16, f32):
    h, w = img.shape
    with open(path, "wb") as f:
        f.write(np.array([w, h], np.int32).tobytes())
        f.write(np.ascontiguousarray(img).tobytes())
        f.write(np.ascontiguousarray(m16[0], np.int16).tobytes())
        f.write(np.ascontiguousarray(m16[1], np.uint16).tobytes())
        f.write(np.ascontiguousarray(f32[0], np.float32).tobytes())
        f.write(np.ascontiguousarray(f32[1], np.float32).tobytes())


def _case(w, h, seed):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (h, w), dtype=np.uint8)
    mx, my = RR.radial_map_np(w, h)
    return img, RR.fixed_from_float(mx, my), (mx, my)


def test_rect_adapter_routes_rectify_image_to_the_device_call(tmp_path):
    """With the device calls mocked (tests/helpers/remap_mock.c: dst = 255 - src): one map creation per calibration however
    many calls, with the map type and the maps' row strides; one ov2_remap per call with the image size, the source's ROI row
    stride, the destination's own stride and one frame; the in-place call hands the same buffer as source and destination and
    gets its result in that buffer; a calibration without maps returns the image itself without a device call."""
    exe = build.build_rect_shim()
    mock = tmp_path / "libmock.so"
    subprocess.check_call(["gcc", "-shared", "-fPIC", "-O1", "-o", str(mock), str(ROOT / "tests" / "helpers" / "remap_mock.c")])
    w, h = 173, 121
    img, m16, f32 = _case(w, h, 5)
    _write_input(tmp_path / "in.bin", img, m16, f32)
    env = dict(os.environ, LD_PRELOAD=str(mock), OV2_MOCK_LOG=str(tmp_path / "log.bin"))
    out = subprocess.run([str(exe), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=60, env=env)
    assert out.returncode == 0, out.stdout + out.stderr
    got = np.fromfile(tmp_path / "out.bin", np.uint8).reshape(4, h, w)
    for k in range(4):
        assert np.array_equal(got[k], 255 - img), k
    log = np.fromfile(tmp_path / "log.bin", np.int32).reshape(-1, 10)
    creates, calls = log[log[:, 0] == 6], log[log[:, 0] == 5]
    assert len(log) == 6 and len(creates) == 2 and len(calls) == 4
    assert creates[0].tolist() == [6, 11, w, h, 4 * w, 2 * w, 0, 0, 0, 0]          # CV_16SC2 + CV_16UC1, created on the first call
    assert creates[1].tolist() == [6, 5, w, h, 4 * w, 4 * w, 0, 0, 0, 0]           # CV_32FC1 x 2
    assert log[0, 0] == 6 and log[3, 0] == 6                                       # the second call of the first map: no new map
    pad = 13
    assert calls[0].tolist() == [5, 11, w, h, w + pad, 0, w, 0, 1, 0]
    assert calls[1].tolist() == [5, 11, w, h, w + pad, 0, w, 0, 1, 0]
    assert calls[2].tolist() == [5, 5, w, h, w, 0, w, 0, 1, 0]
    assert calls[3].tolist() == [5, 11, w, h, w, 0, w, 0, 1, 1]                    # rectifyImage(im0, im0)


def test_rect_shim_compiles_against_the_reference_own_headers():
    """The drop-in translation unit against the reference's include/camera_calibration.hpp (member names undist_map_x_,
    undist_map_y_, intrinsic_mutex_ and the rectifyImage declaration), with stand-ins only for the third-party headers."""
    from oracle.ref_build import check_shims
    if not check_shims.available():
        pytest.skip("/root/reference is not present")
    err = check_shims.check("camera_calibration_rect_gpu.cpp")
    assert not err, err[:3000]


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(752, 480), (333, 217)])
def test_rect_shim_on_the_device_equals_cv2_remap(tmp_path, size):
    """The same self-test with the real library: every rectified image equals cv2.remap (or, where cv2 is absent, remap_ref)
    of the source with the calibration's maps."""
    exe = build.build_rect_shim()
    w, h = size
    img, m16, f32 = _case(w, h, 11)
    _write_input(tmp_path / "in.bin", img, m16, f32)
    out = subprocess.run([str(exe), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    got = np.fromfile(tmp_path / "out.bin", np.uint8).reshape(4, h, w)
    ref = RR.remap_cv2 if RR.cv2 is not None else RR.remap_ref
    want16 = ref(img, *m16)
    assert np.array_equal(got[0], want16) and np.array_equal(got[1], want16) and np.array_equal(got[3], want16)
    assert np.array_equal(got[2], ref(img, *f32))
