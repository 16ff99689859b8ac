"""CPU: the camera model (cph.camera) and geometry.Image as plain data: the accessors of PinholeCameraIntrinsic
(pinhole_camera_intrinsic.h; pybind camera.cpp), PinholeCameraParameters' defaults, and Image's constructor rules
(image.cpp:80-100: uint8, uint16 or float32, 1, 3 or 4 channels).  None of them touches the device."""
import numpy as np
import pytest

import cupoch_b200 as cph

CAM, G = cph.camera, cph.geometry


def test_pinhole_camera_intrinsic():
    c = CAM.PinholeCameraIntrinsic(640, 480, 525.0, 526.0, 319.5, 239.5)
    assert c.width == 640 and c.height == 480 and c.is_valid()
    assert c.get_focal_length() == (525.0, 526.0) and c.get_principal_point() == (319.5, 239.5)
    np.testing.assert_array_equal(c.intrinsic_matrix, np.float32([[525, 0, 319.5], [0, 526, 239.5], [0, 0, 1]]))
    assert c.intrinsic_matrix.dtype == np.float32
    c.set_intrinsics(32, 24, 10, 11, 12, 13)
    assert (c.width, c.height, c.get_focal_length(), c.get_principal_point()) == (32, 24, (10.0, 11.0), (12.0, 13.0))
    c.intrinsic_matrix = np.eye(3) * 2
    assert c.get_focal_length() == (2.0, 2.0) and c.intrinsic_matrix.dtype == np.float32
    assert not CAM.PinholeCameraIntrinsic().is_valid()
    assert not CAM.PinholeCameraIntrinsic(0, 10, 1, 1, 0, 0).is_valid()


def test_pinhole_camera_parameters():
    p = CAM.PinholeCameraParameters()
    assert not p.intrinsic.is_valid()
    np.testing.assert_array_equal(p.extrinsic, np.eye(4, dtype=np.float32))
    p.extrinsic = np.arange(16).reshape(4, 4)
    assert p.extrinsic.dtype == np.float32 and p.extrinsic[3, 2] == 14
    with pytest.raises(ValueError):
        p.extrinsic = np.zeros(9)


@pytest.mark.parametrize("dtype,bpc", [(np.uint8, 1), (np.uint16, 2), (np.float32, 4)])
@pytest.mark.parametrize("shape,ch", [((5, 7), 1), ((5, 7, 1), 1), ((5, 7, 3), 3), ((5, 7, 4), 4)])
def test_image_kinds(dtype, bpc, shape, ch):
    im = G.Image(np.zeros(shape, dtype))
    assert (im.height, im.width, im.num_of_channels, im.bytes_per_channel) == (5, 7, ch, bpc)
    assert not im.is_empty()


@pytest.mark.parametrize("bad", [np.zeros((4, 4), np.float64), np.zeros((4, 4), np.int32), np.zeros((4, 4, 2), np.uint8),
                                 np.zeros((4, 4, 5), np.float32), np.zeros(4, np.uint8), np.zeros((2, 2, 2, 1), np.uint8)])
def test_image_rejects(bad):
    with pytest.raises(ValueError):
        G.Image(bad)
