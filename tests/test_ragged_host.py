"""CPU: the host side of the ragged uint8 forward (i2it_forward with x_u8_list).  A dimension that does not change is an identity
pass whose bytes equal PIL skipping it; the descriptor tables a call uploads fit the area its plan reserves; the wrappers'
geometry lists and the default capacity."""
import numpy as np
import pytest

import pil_resample as R


def _identity_pass(img, axis):
    """pil_resample's pass arithmetic with the one-tap table the ragged passes use for an unchanged dimension."""
    n = img.shape[axis]
    x = np.moveaxis(img, axis, 0).astype(np.int64)
    acc = np.full(x.shape, 1 << (R.PRECISION_BITS - 1), np.int64) + (1 << R.PRECISION_BITS) * x[np.arange(n)]
    return np.ascontiguousarray(np.moveaxis(np.clip(acc >> R.PRECISION_BITS, 0, 255).astype(np.uint8), 0, axis))


@pytest.mark.parametrize("n", [1, 2, 7, 64, 517, 4032])
def test_unchanged_dimension_table_is_the_identity(n):
    """The library's own (n -> n) table has one tap of 1 << 22 at each output's own index and zeros elsewhere: the one-tap
    identity table of the ragged passes is what PIL's arithmetic would compute for a pass it skips."""
    import i2it
    ksize, bounds, coeffs = i2it.resample_coeffs(n, n)
    rk, rb, rc = R.coeffs(n, n)
    assert ksize == rk and bounds == [tuple(b) for b in rb.tolist()] and coeffs == rc.tolist()
    for i, ((xmin, taps), k) in enumerate(zip(bounds, coeffs)):
        nz = [(xmin + t, c) for t, c in enumerate(k[:taps]) if c != 0]
        assert nz == [(i, 1 << R.PRECISION_BITS)], (i, nz)
        assert all(c == 0 for c in k[taps:])


def test_identity_weight_keeps_every_byte():
    v = np.arange(256, dtype=np.int64)
    assert np.array_equal(((1 << 21) + v * (1 << 22)) >> 22, v)


@pytest.mark.parametrize("src,dst", [((40, 50), (61, 50)), ((97, 131), (97, 128)), ((9, 300), (1, 300)), ((33, 21), (33, 21))])
def test_identity_pass_equals_pil_skipping_it(src, dst):
    """Both passes always run in the ragged path: the identity one leaves PIL's bytes."""
    img = R.stripe_image(*src, seed=src[0] * src[1])
    x = img[None]
    x = R._pass(x, 2, dst[1]) if src[1] != dst[1] else _identity_pass(x, 2)
    x = R._pass(x, 1, dst[0]) if src[0] != dst[0] else _identity_pass(x, 1)
    assert np.array_equal(x[0], R.pil_resize(img, dst))


FRAMES = [(480 + round(i * 600 / 23), 640 + round(i * 1280 / 23)) for i in range(24)]
SWEEP = FRAMES + [(1, 1), (3024, 4032), (4032, 3024), (512, 512), (7, 4096), (4096, 7), (333, 517), (64, 90)]


@pytest.mark.parametrize("prep", ["resize_512x512", "resized_crop_512", "resize_256x256"])
@pytest.mark.parametrize("slack", [0, 3000])
def test_table_bound_holds(prep, slack):
    """Every image of the sweep, alone and all together, uploads no more table ints than the plan's bound reserves, at the
    default capacity and above it."""
    import i2it
    from _host import ragged_geometries
    H, W, geoms = ragged_geometries(SWEEP, image_prep=prep)
    cap = i2it.ragged_max_side([v for g in geoms for v in g["resize"] + g["out_size"]]) + slack
    for hw, g in zip(SWEEP, geoms):
        used, bound = i2it.ragged_table_ints([g], [hw], cap)
        assert 0 < used <= bound, (hw, used, bound)
    used, bound = i2it.ragged_table_ints(geoms, SWEEP, cap)
    assert 0 < used <= bound


def test_table_bound_at_extremes():
    """The bound's worst cases: downscaling from max_side to a 8-pixel network and upscaling back, identity at max_side."""
    import i2it
    for ms in (8, 64, 4096, 5120):
        for hw, net in [((ms, ms), (8, 8)), ((ms, 1), (8, 8)), ((1, ms), (8, 8)), ((8, 8), (8, 8))]:
            g = {"resize": net, "out_size": hw}
            used, bound = i2it.ragged_table_ints([g], [hw], ms)
            assert used <= bound, (ms, hw, used, bound)
        g = {"resize": (ms, ms), "crop": (0, 0, 8, 8), "out_size": (ms, ms)}
        used, bound = i2it.ragged_table_ints([g], [(ms, ms)], ms)
        assert used <= bound


def test_host_sizing_rejects_bad_geometry():
    import i2it
    with pytest.raises(ValueError, match="reject"):
        i2it.ragged_table_ints([{"resize": (512, 512)}], [(5000, 300)], 4096)          # above max_side
    with pytest.raises(ValueError, match="reject"):
        i2it.ragged_table_ints([{"resize": (512, 512), "crop": (1, 0, 512, 512)}], [(600, 300)], 4096)   # crop outside
    with pytest.raises(ValueError, match="one network size"):
        i2it.ragged_table_ints([{"resize": (512, 512)}, {"resize": (256, 256)}], [(600, 300), (600, 300)], 4096)


def test_max_side_rounding():
    import i2it
    assert i2it.ragged_max_side([1, 512]) == 4096
    assert i2it.ragged_max_side([4096]) == 4096
    assert i2it.ragged_max_side([4097]) == 5120
    assert i2it.ragged_max_side([720, 1280, 5121]) == 6144
    assert i2it.ragged_max_side([2 ** 14]) == 2 ** 14


def test_wrapper_geometries():
    from _host import image_prep_geometry, ragged_geometries
    sizes = [(720, 1280), (1080, 1920), (333, 517), (512, 512)]
    H, W, g = ragged_geometries(sizes, image_prep="resize_512x512")
    assert (H, W) == (512, 512)
    assert g == [{"resize": (512, 512), "crop": None, "out_size": hw} for hw in sizes]
    H, W, g = ragged_geometries(sizes, image_prep="resized_crop_512")
    assert (H, W) == (512, 512)
    for hw, d in zip(sizes, g):
        rs, crop = image_prep_geometry("resized_crop_512", *hw)
        assert d == {"resize": rs, "crop": crop, "out_size": hw}
    H, W, g = ragged_geometries(sizes, resize=(256, 384))
    assert (H, W) == (256, 384) and all(d["resize"] == (256, 384) and d["out_size"] == hw for hw, d in zip(sizes, g))
    with pytest.raises(ValueError, match="one network size"):
        ragged_geometries(sizes, image_prep="no_resize")
    with pytest.raises(ValueError, match="random crops"):
        ragged_geometries(sizes, image_prep="randomcrop_hflip")
    with pytest.raises(ValueError, match="at least one"):
        ragged_geometries([], image_prep="resize_512x512")
