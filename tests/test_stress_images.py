"""The adversarial image set of tests/stress_images.py is deterministic: the GPU tests and the reference's stored runs
(tests/golden/live/stress_*.npz, knob_*.npz) were made from exactly these bytes."""
import hashlib

import numpy as np
import pytest

import stress_images as si

SHA256 = {
    "checker_p2": "6924c1ba06fb23d0ab028279f5f8e598e51448768496a99ef102562912ce9283",
    "checker_p3": "e8819537274c964ab28fa519084871a1f71fdd82079a3a5a4cf83f1872bf35ca",
    "checker_p8": "3cf0bedb9f1963924338b92261cbf243ff6549a5af07e1e73709c17ae07c934f",
    "checker_rot30_p6": "56f193f6a8efcb6552b92ac4fef7f875d56fd59cd108c7d741bcca5fafb9088c",
    "block_noise_4": "55583effe649b2862d9abb092308f3318da9d63f9db4ec36b87532381449e95d",
    "binary_noise": "d03715615e81280d3c988d293c381fda359089a485b9552e833705377c3ce424",
    "saturated": "f69e00b79aa1f0cce9d6575ab6f2702abf8ee2678d284e191d00a9d74993e0ed",
    "dark": "d8cf2483a07ee82219276215f5c0a1d6ec484121f62bb739f6119bac63ebdd9e",
    "border_impulses": "b8ab9eeb6ca60b0c4b68752a1ac899d1769fe7fd4ce860d72c644af275ef1882",
    "step_edges": "e568b97900286b25682df504a98257c3c45db1ddde0e0cd4edb69dadcbf19b58",
    "const_0": "17744bb6a4ed1d9d51d85d7eb645cde30352530d494233c434027f9e3193bae4",
    "const_255": "bd720a5704fa8160ef0a7dc2e31c155e89d6a314b3b0fec0f52f5cb8075381c6",
    "binary_noise_f32": "bcc33cdbc7030409787a894e9006ec53a9128c27b4b6b7e4414591a986df8d4f",
    "checker_p8_f32": "df943fac9388aef40819f34838e411628548bfeef6fff9951ae0863eed93922a",
    "checker_p3_4k": "aa3136cdd570082b075bb963e8f1ddea3a6d3b33e5848dc6a762dd13c0824d11",
}


def test_every_image_is_pinned():
    assert sorted(SHA256) == sorted(si.NAMES)


@pytest.mark.parametrize("name", sorted(SHA256))
def test_stress_image_bytes_are_pinned(name):
    a = si.image(name)
    assert a.shape == si.SIZES[name][::-1]
    assert hashlib.sha256(a.tobytes()).hexdigest() == SHA256[name]
    assert np.array_equal(a, si.image(name))                          # same name, same bytes
    if a.dtype == np.float32:
        assert set(np.unique(a).tolist()) == {0.0, 1.0}               # the top of the FloatImages range, exactly
    else:
        assert a.dtype == np.uint8


def test_full_contrast_images_use_only_0_and_255():
    for name in ("checker_p2", "checker_p3", "checker_p8", "checker_rot30_p6", "block_noise_4", "binary_noise", "step_edges"):
        assert set(np.unique(si.image(name)).tolist()) == {0, 255}, name
    assert set(np.unique(si.image("dark")).tolist()) == {0, 1, 2, 3}
    b = si.image("border_impulses")
    for edge in (b[0], b[-1], b[:, 0], b[:, -1], b[1], b[-2], b[:, 1], b[:, -2]):   # structure in the outermost rows / columns
        assert (edge == 0).any() and (edge == 255).any()


def test_other_sizes_keep_the_content():
    a = si.image("block_noise_4", 97, 61)
    assert a.shape == (61, 97) and np.array_equal(si.image("checker_p8", 97, 61), si.image("checker_p8")[:61, :97])
