"""CPU: the LANCZOS resize restatement (tests/pil_resample.py) equals PIL bit for bit, the library's host coefficient tables
equal the restatement's, and image_prep_geometry equals what torchvision's Resize / CenterCrop do to PIL images."""
import random

import numpy as np
import pytest

import pil_resample as R

SHAPES = [   # (H, W) -> (H2, W2)
    ((720, 1280), (512, 512)), ((512, 512), (720, 1280)), ((517, 333), (512, 328)), ((300, 200), (256, 256)),
    ((64, 96), (286, 286)), ((1000, 37), (8, 512)), ((97, 131), (97, 128)), ((3024, 504), (512, 40)),
    ((1, 1), (5, 7)), ((1, 9), (300, 1)), ((9, 300), (1, 1)), ((40, 50), (40, 77)), ((40, 50), (61, 50)),
    ((40, 50), (40, 50)), ((3024, 4032), (512, 512)), ((512, 512), (3024, 4032)),
]


@pytest.mark.parametrize("src,dst", SHAPES, ids=[f"{a[0]}x{a[1]}-{b[0]}x{b[1]}" for a, b in SHAPES])
def test_restatement_equals_pil(src, dst):
    img = R.stripe_image(*src, seed=src[0] * 7 + dst[1])
    got = R.resize(img, dst)
    ref = R.pil_resize(img, dst)
    assert got.shape == ref.shape == dst + (3,)
    assert (got != ref).sum() == 0


def test_restatement_batch_is_per_image():
    imgs = R.stripe_image(45, 70, seed=5, b=3)
    got = R.resize(imgs, (32, 101))
    for i in range(3):
        assert np.array_equal(got[i], R.pil_resize(imgs[i], (32, 101)))


def _pairs():
    rng = random.Random(0)
    pairs = [(1, 1), (1, 512), (512, 1), (4032, 512), (512, 4032), (3024, 512), (720, 512), (1280, 512), (512, 720),
             (512, 1280), (1080, 512), (1920, 512), (512, 1080), (512, 1920), (333, 328), (517, 512), (131, 128), (7, 7)]
    pairs += [(rng.randint(1, 1100), rng.randint(1, 1100)) for _ in range(260)]
    pairs += [(rng.randint(1, 40), rng.randint(1, 2000)) for _ in range(20)]
    return pairs


def test_library_tables_equal_restatement():
    import i2it
    worst = 0.0
    for a, b in _pairs():
        ks, bounds, kk = i2it.resample_coeffs(a, b)
        rks, rb, rk = R.coeffs(a, b)
        assert ks == rks, (a, b)
        assert np.array_equal(np.array(bounds, np.int32), rb), (a, b)
        assert np.array_equal(np.array(kk, np.int32), rk), (a, b)
        worst = max(worst, float(np.abs(rk.astype(np.int64)).sum(1).max()))
    # the int32 argument of csrc/resample.cuh: 2^21 + 255 * sum|k| < 2^31 with room to spare
    assert 2 ** 21 + 255 * worst < 0.8 * 2 ** 31, worst


def test_library_refuses_bad_sizes():
    import i2it
    lib = i2it.load_library()
    assert lib.i2it_debug_resample_coeffs(0, 5, None, None, 0) == -1
    assert lib.i2it_debug_resample_coeffs(5, -1, None, None, 0) == -1
    ks = lib.i2it_debug_resample_coeffs(100, 10, None, None, 0)
    import ctypes as C
    buf = (C.c_int * (10 * ks - 1))()
    assert lib.i2it_debug_resample_coeffs(100, 10, None, buf, 10 * ks - 1) == -1      # short coefficient buffer


SIZES = [(720, 1280), (1280, 720), (1080, 1920), (3024, 4032), (512, 512), (512, 768), (333, 517), (600, 601), (97, 131),
         (513, 512)]


@pytest.mark.parametrize("prep", ["resize_512x512", "resize_512", "resize_256x256", "resize_256", "resized_crop_512",
                                  "no_resize"])
def test_image_prep_geometry_matches_torchvision(prep):
    from PIL import Image
    from torchvision import transforms
    from _host import image_prep_geometry
    T = {
        "resized_crop_512": transforms.Compose([transforms.Resize(512, interpolation=transforms.InterpolationMode.LANCZOS),
                                                transforms.CenterCrop(512)]),
        "resize_256": transforms.Resize((256, 256), interpolation=Image.LANCZOS),
        "resize_256x256": transforms.Resize((256, 256), interpolation=Image.LANCZOS),
        "resize_512": transforms.Resize((512, 512), interpolation=Image.LANCZOS),
        "resize_512x512": transforms.Resize((512, 512), interpolation=Image.LANCZOS),
        "no_resize": transforms.Lambda(lambda x: x),
    }[prep]
    for H, W in SIZES:
        img = R.stripe_image(H, W, seed=H + W)
        ref = np.asarray(T(Image.fromarray(img)))
        rs, crop = image_prep_geometry(prep, H, W)
        got = R.resize(img, rs)
        if crop is not None:
            top, left, h, w = crop
            assert 0 <= top and top + h <= rs[0] and 0 <= left and left + w <= rs[1]
            got = got[top:top + h, left:left + w]
        assert got.shape == ref.shape and np.array_equal(got, ref), (prep, H, W, rs, crop)


def test_image_prep_geometry_rejects_random_crops():
    from _host import image_prep_geometry
    with pytest.raises(ValueError):
        image_prep_geometry("resize_286_randomcrop_256x256_hflip", 720, 1280)
    with pytest.raises(ValueError):
        image_prep_geometry("resize_1024", 720, 1280)


def test_paired_geometry_is_the_cli_rule():
    from _host import paired_geometry
    assert paired_geometry(721, 1283) == (720, 1280)
    assert paired_geometry(512, 512) == (512, 512)
