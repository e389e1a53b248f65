"""CPU checks of the point-cloud Node-constructor oracle (tests/cloud_oracle.py) and of the flags that select it: the colour
conversion against cv2 on every RGB triple, calculateDepthMask against the C++ cast it restates, and, on rendered frames,
how often the reference's compute() would separate descriptors from their 3-D points."""
import re
import subprocess
from pathlib import Path

import cv2
import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent

MASK_SRC = r"""
#include <cstdio>
#include <vector>
int main(int argc, char** argv) {  // float32 values in, one calculateDepthMask byte per value out
  std::FILE* f = std::fopen(argv[1], "rb");
  std::vector<float> v;
  float x;
  while (std::fread(&x, 4, 1, f) == 1) v.push_back(x);
  std::fclose(f);
  std::vector<unsigned char> out(v.size());
  for (size_t i = 0; i < v.size(); i++) {
    volatile float value = v[i];
    out[i] = value != value ? 0 : static_cast<unsigned char>(value * 50.0);  // openni_listener.cpp:520-534
  }
  f = std::fopen(argv[2], "wb");
  std::fwrite(out.data(), 1, out.size(), f);
  std::fclose(f);
  return 0;
}
"""


def test_rgb_to_gray_matches_cv2_on_all_triples():
    import cloud_oracle as co
    a = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.stack([(a >> 16) & 255, (a >> 8) & 255, a & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    assert np.array_equal(co.rgb_to_gray(rgb), cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY))
    # channel 0 is R: a bgr8 image is converted with R and B swapped, as the reference's CV_RGB2GRAY does
    px = np.array([[[200, 10, 10], [10, 10, 200]]], np.uint8)
    assert co.rgb_to_gray(px).tolist() == [[67, 32]]


def test_cloud_mask_matches_the_cpp_cast(tmp_path):
    import platform

    import cloud_oracle as co
    if platform.machine() not in ("x86_64", "AMD64"):
        pytest.skip("the restated out-of-range behaviour is x86-64's cvttsd2si")
    src = tmp_path / "mask.cpp"
    src.write_text(MASK_SRC)
    exe = tmp_path / "mask"
    subprocess.run(["g++", "-O2", str(src), "-o", str(exe)], check=True)
    special = [0.0, -0.0, 0.0199, 0.02, 0.0201, 1.0, 5.11, 5.12, 5.1201, 5.13, 6.0, 10.24, 10.25, 42.9, 1e3, 4.29e7, 4.3e7, 1e8, 1e30,
               np.inf, -np.inf, np.nan, -0.01, -0.02, -0.03, -1.0, -5.12, -5.13, -4.29e7, -4.3e7, -1e8, -np.inf]
    rng = np.random.default_rng(0)
    z = np.concatenate([np.array(special, np.float32), np.linspace(-12, 12, 200001, dtype=np.float32),
                        rng.uniform(-1e9, 1e9, 10000).astype(np.float32), np.float32(10.0) ** rng.uniform(-3, 12, 10000).astype(np.float32)])
    (tmp_path / "z.bin").write_bytes(z.tobytes())
    subprocess.run([str(exe), str(tmp_path / "z.bin"), str(tmp_path / "m.bin")], check=True)
    ref = np.frombuffer((tmp_path / "m.bin").read_bytes(), np.uint8)
    assert np.array_equal(co.cloud_mask(z), ref)
    # the values the header and DESIGN quote
    got = dict(zip(special, co.cloud_mask(np.array(special, np.float32)).tolist()))
    assert got[0.02] == 0 and got[5.12] == 255 and got[5.13] == 0 and got[6.0] == 44 and got[1e8] == 0 and got[np.inf] == 0
    assert got[-1.0] == 206  # negative depths wrap too


@pytest.fixture(scope="module")
def rendered():
    from rgbdslam_v2_b200 import synth
    poses = synth.trajectory(40)
    return [synth.render_frame(poses[k], seed=k) for k in (0, 5, 10)]


@pytest.mark.parametrize("detector", ["ORB", "FAST"])
def test_reference_compute_separates_points_from_descriptors(rendered, detector):
    """In the reference, compute() runs after projectTo3D and drops / re-orders the 2-D keypoints but not the 3-D points.
    Count, on rendered frames, the node rows whose point would belong to another keypoint: that is routine, not rare."""
    import cloud_oracle as co
    from oracle import orb_oracle as oo
    from rgbdslam_v2_b200 import synth
    K4 = (synth.FX, synth.FY, synth.CX, synth.CY)
    st = oo.DetectorState()
    mismatched = dropped = 0
    for gray, depth in rendered:
        cloud = co.cloud_from_depth(depth, K4)
        rec = co.detect(gray, oo.depth_to_mask(depth), st, 600, detector=detector)
        kept, pts = co.project_to_3d(rec, cloud, 600)
        kp, desc, src = co.compute_tracked(gray, kept)
        assert len(kp) == len(desc) <= len(kept) == len(pts) <= 600
        dropped += len(kept) - len(kp)
        # row i of the reference node: descriptor of keypoint src[i], point of keypoint i
        mismatched += int((src != np.arange(len(src))).sum())
        # the library's node keeps them together: its point of row i is that of keypoint src[i]
        k2, d2, xyz = co.node_construct(gray, cloud, oo.depth_to_mask(depth), oo.DetectorState(), 600, detector=detector)
        assert len(k2) > 0 and np.isfinite(xyz[:, 3]).all()
    assert dropped > 0 and mismatched > 100, (dropped, mismatched)


def _header_defines():
    txt = (ROOT / "include" / "rgbdslam_b200.h").read_text()
    return {m.group(1): int(m.group(2)) for m in re.finditer(r"#define RGBDSLAM_B200_(\w+) (\d+)\b", txt)}


def test_flag_constants_and_capi_mirror():
    from rgbdslam_v2_b200 import _capi
    d = _header_defines()
    assert d["MASK_FROM_DEPTH"] == _capi.MASK_FROM_DEPTH == 1
    assert d["VISUAL_RGB"] == _capi.VISUAL_RGB == 2
    assert d["CLOUD_XYZRGB"] == _capi.CLOUD_XYZRGB == 4
    assert d["CLOUD_XYZ"] == _capi.CLOUD_XYZ == 8
    assert d["MASK_FROM_CLOUD"] == _capi.MASK_FROM_CLOUD == 16
    f = _capi.node_input_flags
    assert f((2, 48, 64), (2, 48, 64)) == 0
    assert f((2, 48, 64), (2, 48, 64), mask_from_depth=True) == _capi.MASK_FROM_DEPTH
    assert f((2, 48, 64, 3), (2, 48, 64)) == _capi.VISUAL_RGB
    assert f((2, 48, 64), (2, 48, 64, 8)) == _capi.CLOUD_XYZRGB
    assert f((2, 48, 64, 3), (2, 48, 64, 4), mask_from_cloud=True) == _capi.VISUAL_RGB | _capi.CLOUD_XYZ | _capi.MASK_FROM_CLOUD
    for g, dshape in (((2, 48, 64, 4), (2, 48, 64)), ((2, 48, 64), (2, 48, 64, 3))):
        with pytest.raises(ValueError):
            f(g, dshape)
