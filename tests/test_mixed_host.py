"""CPU: the host side of the mixed-direction CycleGAN forward (i2it_forward with directions).  The new symbols are exported,
the request descriptors have the C layout, the wrappers validate direction and caption lists before anything reaches the
engine, and the size rule holds at its boundaries."""
import ctypes as C
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["i2it_mixed_size_check", "i2it_op_conv2d_sel"]


def test_mixed_symbols_are_exported_and_typed():
    import i2it
    lib = i2it.load_library()
    for s in NEW_SYMBOLS:
        assert s in i2it.SYMBOLS
        fn = getattr(lib, s)
        assert fn.argtypes is not None and fn.restype is C.c_int, s
    assert len(lib.i2it_op_conv2d_sel.argtypes) == 7


def test_struct_layouts_match_ctypes(tmp_path):
    """sizeof, and every field's offsetof and size, of the structs include/i2it.h declares, as the host C compiler lays them
    out, equal the ctypes mirrors'.  A mismatch would hand the library shifted fields without any error."""
    import i2it
    structs = {"i2it_forward_desc": i2it.ForwardDesc, "i2it_resize_desc": i2it.ResizeDesc, "i2it_conv_desc": i2it.ConvDesc,
               "i2it_config": i2it.Config, "i2it_memory_stats": i2it.MemoryStats}
    lines, want = [], []
    for name, cls in structs.items():
        lines.append(f'printf("{name} %zu\\n", sizeof({name}));')
        want.append(f"{name} {C.sizeof(cls)}")
        for f, _ in cls._fields_:
            lines.append(f'printf("{name}.{f} %zu %zu\\n", offsetof({name}, {f}), sizeof((({name}*)0)->{f}));')
            want.append(f"{name}.{f} {getattr(cls, f).offset} {getattr(cls, f).size}")
    src = tmp_path / "layout.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"i2it.h\"\nint main(void) {\n" + "\n".join(lines) +
                   "\nreturn 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")[:-1]
    assert got == want


@pytest.mark.parametrize("H,W", [(512, 512), (256, 256), (512, 768), (768, 512), (1024, 1024), (128, 128), (64, 128)])
def test_accepted_sizes(H, W):
    import i2it
    assert i2it.mixed_size_check(H, W) == ""


def test_token_rule_refuses_1280x720():
    """(720/8)(1280/8) = 14400 latent pixels = 112.5 tiles of 128 rows: a token tile would hold rows of two images."""
    import i2it
    for H, W in ((720, 1280), (1280, 720)):
        why = i2it.mixed_size_check(H, W)
        assert "multiple of 128" in why and "14400" in why, why


@pytest.mark.parametrize("H,W,ok", [
    (64, 128, True),      # latent 8 x 16 = 128 tokens; the 16 x 8 box of the latent convs fills 128 pixels of one image
    (32, 256, False),     # latent 4 x 32 = 128 tokens, but a 16 x 4 box spans two images
    (64, 64, False),      # latent 8 x 8: an 8 x 8 box spans two images (and 64 tokens)
    (8, 1024, False),     # latent 1 x 128: the stride-2 conv into it has a 16 x 1 box
    (64, 256, True),
    (48, 256, False),     # latent 6 x 32 = 192 tokens: not a multiple of 128
])
def test_tile_box_rule_at_its_boundary(H, W, ok):
    import i2it
    why = i2it.mixed_size_check(H, W)
    assert (why == "") == ok, why
    if not ok and (H // 8) * (W // 8) % 128 == 0:
        assert "tile box" in why and "images" in why, why


def test_size_rule_follows_the_conv_box_picker():
    """Sweep: a size is accepted iff its token count is a multiple of 128 and every level's box (the picker's formula,
    restated) covers 128 pixels of one image."""
    import i2it

    def p2(v):
        p = 1
        while p < v:
            p *= 2
        return p

    def one_image(h, w, s1, cap):
        tw = min(128, p2(w)) if (s1 and h == 1) else min(cap, p2(w))
        th = min(128 // tw, p2(h))
        return tw * th == 128

    for H in range(8, 264, 8):
        for W in (8, 64, 128, 136, 256, 1024):
            ok = (H // 8) * (W // 8) % 128 == 0
            for k in range(4):
                h, w = H >> k, W >> k
                ok = ok and one_image(h, w, True, 16) and (k > 0 or one_image(h, w, True, 32))
                ok = ok and (k == 0 or one_image(h, w, False, 16))
            assert (i2it.mixed_size_check(H, W) == "") == ok, (H, W)


def test_size_check_rejects_non_multiples_of_8():
    import i2it
    assert "multiples of 8" in i2it.mixed_size_check(100, 512)


@pytest.mark.parametrize("dirs,msg", [
    ([0, 1], "3 images but 2 directions"),
    ([0, 2, 1], "direction 2 of image 1"),
    ([0, True, 1], "direction True of image 1"),
    ([0, "b2a", 1], "direction 'b2a' of image 1"),
])
def test_engine_direction_array_validation(dirs, msg):
    import i2it
    with pytest.raises(ValueError, match=msg):
        i2it.directions_array(dirs, 3)


def test_engine_direction_array():
    import i2it
    a = i2it.directions_array([i2it.A2B, i2it.B2A, i2it.B2A], 3)
    assert list(a) == [0, 1, 1]


def test_wrapper_direction_codes():
    import i2it
    from cyclegan_turbo import direction_codes
    assert direction_codes("a2b", 4) == i2it.A2B and direction_codes("b2a", 4) == i2it.B2A
    assert direction_codes(["a2b", "b2a", "b2a"], 3) == [i2it.A2B, i2it.B2A, i2it.B2A]
    assert direction_codes(("b2a",), 1) == [i2it.B2A]
    with pytest.raises(ValueError, match="2 images but 3 directions"):
        direction_codes(["a2b", "b2a", "a2b"], 2)
    with pytest.raises(ValueError, match="neither 'a2b' nor 'b2a'"):
        direction_codes(["a2b", "A2B"], 2)
    with pytest.raises(ValueError, match="neither 'a2b' nor 'b2a'"):
        direction_codes(["a2b", 1], 2)
    with pytest.raises(ValueError, match="direction must be"):
        direction_codes("c2d", 1)
    with pytest.raises(ValueError, match="direction must be"):
        direction_codes(1, 1)


def test_wrapper_caption_lists():
    from cyclegan_turbo import check_caption
    assert check_caption("night", 3) == "night"
    assert check_caption(["a", "b"], 2) == ["a", "b"]
    assert check_caption(("a", "b"), 2) == ["a", "b"]
    with pytest.raises(ValueError, match="2 images but 3 captions"):
        check_caption(["a", "b", "c"], 2)
    with pytest.raises(ValueError, match="string or a list of strings"):
        check_caption(["a", 3], 2)
    with pytest.raises(ValueError, match="string or a list of strings"):
        check_caption(None, 2)
