"""tapgemm conformance matrix: every kernel instantiation (dtype x lean/full x BN) held to the float64 bound of tests/kref.py at
forced tile widths, ring depths and persistent grids (i2it_debug_tapgemm_override), so a configuration is reached on purpose
and not only when pick_bn happens to choose it for a test shape on the card the suite runs on.

For a fixed GEMM, BN, ring depth, grid, store boxes (I2IT_NO_OSTG2) and epilogue variant (I2IT_NO_LEAN) change data movement
only (DESIGN section 6), so every configuration of one op must give the bits of the engine's own choice; GroupNorm outputs
must agree among the runs that share a statistics path (epilogue partials or the statistics pass).

Each sub-case is asserted, from the launch strings, to have run with the forced BN / st / grid and the expected lean / tma /
tma2 / gn.  The sub-cases of one instantiation include several tiles per CTA with a grid that does not divide the n-tile count
(the CTA's n-tile changes from one tile to the next, so its bias slice is restaged), ragged last n-tiles, m-tiles that span
images with partial edges, token rows that are not a multiple of 128, K tails (Cin = 8, 72), a 3x3 conv with more than 48
k-steps, a ring of 2 stages and one of (k-steps - 1) stages, and every epilogue the width can run.

test_production_signatures_are_covered runs the BASELINE configs (#2, #4, #5's batches 1 ... 16) on random SD-Turbo-size
weights and checks that every
(dtype, variant, BN, store mode, gn, several tiles per CTA) signature their tapgemm launches use is one the matrix declares
(SIGNATURE_MODES) and exercises.  The CPU test at the end keeps the matrix's instantiation list equal to the engine's."""
import math
import os
import re
import time

import pytest
import torch

import kref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
bf, hf = torch.bfloat16, torch.float16
DTYPE_NAME = {bf: "bf16", hf: "fp16"}

# the instantiations of csrc/engine.cu (TG_BN_LEAN, TG_BN_FULL)
BN_LEAN = (64, 128, 192, 256)
BN_FULL = (16, 32, 48, 64, 80, 96, 112, 128, 160, 192, 224, 256)
INSTANTIATIONS = [("lean", n) for n in BN_LEAN] + [("full", n) for n in BN_FULL]

# Store modes each instantiation runs with in the matrix.  Every mode is run with one tile per CTA and with several, the TMA
# modes with and without GroupNorm statistics from the epilogue.  BN = 256 never gets the second store box (tma2): its four
# ring stages leave no 32 KB to spare.
SIGNATURE_MODES = {
    ("lean", 64): ("tma", "tma2"), ("lean", 128): ("tma", "tma2"), ("lean", 192): ("tma", "tma2"), ("lean", 256): ("tma",),
    **{("full", n): ("direct",) for n in (16, 32, 48, 80, 96, 112, 160, 224)},
    ("full", 64): ("direct", "tma", "tma2"), ("full", 128): ("direct", "tma", "tma2"), ("full", 192): ("direct", "tma", "tma2"),
    ("full", 256): ("direct", "tma"),
}


def declared_signatures(dtype, variant, bn):
    return {(DTYPE_NAME[dtype], variant, bn, mode, gn, multi) for mode in SIGNATURE_MODES[(variant, bn)]
            for gn in ((False,) if mode == "direct" else (False, True)) for multi in (False, True)}


def parse_launch(kind, shape):
    """A tapgemm launch string -> its fields and flags."""
    f = dict(re.findall(r"(\w+)=(\S+)", shape))
    flags = set(shape.split())
    return {"kind": kind, "shape": shape, "BN": int(f["BN"]), "N": int(f["N"]), "tiles": int(f["tiles"]), "grid": int(f["grid"]),
            "st": int(f["st"]), "mode": "tma2" if "tma2" in flags else ("tma" if "tma" in flags else "direct"),
            "gn": "gn" in flags, "lean": "lean" in flags}


def signature(dtype, g):
    return (DTYPE_NAME[dtype], "lean" if g["lean"] else "full", g["BN"], g["mode"], g["gn"], g["tiles"] > g["grid"])


def tapgemm_launches(ops):
    return [parse_launch(o["kind"], o["shape"]) for o in ops if o["kind"].startswith("tapgemm:")]


# ---------------------------------------------------------------------------------------------------------------------
# operands and sub-cases
# ---------------------------------------------------------------------------------------------------------------------
def mk(*shape, dtype=torch.float32, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(dtype)


def weight(Cout, Cin, k, dtype, seed):
    """fp32 weights exactly representable in the engine dtype (the fold rounds nothing)."""
    return mk(Cout, Cin, k, k, scale=1 / math.sqrt(Cin * k * k), seed=seed).to(dtype).float()


def nchw(t):
    return t.double().permute(0, 3, 1, 2)


def predicted_tma2(bn, ksteps):
    """launch_gemm's second store box: K short enough and four stages left after taking 32 KB from the 192 KB ring."""
    per = 16384 + (bn * 128 + 1023) // 1024 * 1024
    return ksteps <= 48 and (4 * 49152 - 32768) // per >= 4


class Sub:
    """One op: how to call it, its float64 check, and what its main tapgemm launch must look like."""

    def __init__(self, name, call, check, *, main, ksteps, tma, gn=False, act=0, engines=("default",), fixed_bn=None,
                 must=()):
        self.name, self.call, self.check, self.main, self.ksteps = name, call, check, main, ksteps
        self.tma, self.gn, self.act, self.engines, self.fixed_bn, self.must = tma, gn, act, engines, fixed_bn, must


def conv_sub(dtype, bn, name, N, H, W, Cin, Cout, k=3, *, res=False, act=0, C2=0, tokens=False, gn=False, out_fp32=False,
             up2x=False, engines=("default",), seed=0):
    import i2it
    geglu = act == i2it.ACT_GEGLU
    oc = Cout // 2 if geglu else Cout
    Ho, Wo = (2 * H, 2 * W) if up2x else (H, W)
    x = mk(N, H, W, Cin, dtype=dtype, seed=seed + 1)
    w = mk(Cout, Cin, 3, 3, scale=1 / math.sqrt(9 * Cin), seed=seed + 2) if up2x else weight(Cout, Cin, k, dtype, seed + 2)
    b = mk(Cout, seed=seed + 3) * 0.5                  # a different bias per column: a stale bias slice shows
    r = mk(N, Ho, Wo, oc, dtype=dtype, seed=seed + 4) if res else None
    x2 = mk(N, Ho, Wo, C2, dtype=dtype, seed=seed + 5) if C2 else None
    w2 = weight(Cout, C2, 1, dtype, seed + 6) if C2 else None
    gamma, beta = mk(oc, seed=seed + 7) * 0.2 + 1, mk(oc, seed=seed + 8) * 0.1
    gnp = (gamma, beta, 1e-6, True) if gn else None
    if up2x:
        wsub = kref.subpixel_weights(w, dtype)
        ref, mag, K = kref.subpixel_conv64(x, wsub, b), kref.subpixel_conv64(x.abs(), wsub.abs(), b.abs()), 4 * Cin
    else:
        ref, mag, K = kref.conv64(x, w, b), kref.conv64(x.abs(), w.abs(), b.abs()), Cin * k * k
    if C2:
        ref, mag, K = ref + kref.conv64(x2, w2), mag + kref.conv64(x2.abs(), w2.abs()), K + C2
    factor = 1.0
    if geglu:
        h, gg = ref.chunk(2, dim=1)
        mh, mg = mag.chunk(2, dim=1)
        ref, mag, factor = h * kref.gelu64(gg), mh * kref.gelu64(gg).abs() + h.abs() * mg, 2.0
    elif act in (i2it.ACT_GELU, i2it.ACT_QUICKGELU):
        ref = kref.gelu64(ref) if act == i2it.ACT_GELU else kref.quick_gelu64(ref)
        factor = 2.0
    if res:
        ref, mag = ref + nchw(r), mag + nchw(r).abs()
    if act == i2it.ACT_CLAMP1:
        ref = ref.clamp(-1, 1)
    # the GEGLU interleave (h_j, gate_j) travels in pairs, so the prepared weight is the same tensor however it is tiled
    acols = 128 if geglu else 64
    tma = not out_fp32 and Cout % acols == 0 and bn % acols == 0 and not (geglu and res)

    def call(E):
        y = E.op_conv2d_ex(x, w, b, residual=r, act=act, x2=x2, w2=w2, up2x=up2x, tokens=tokens, gn=gnp, out_fp32=out_fp32)
        return y if gn else (y, None)

    def check(y, g):
        cs = [kref.check_gemm(name, nchw(y), ref, mag, K, dtype, factor, out_fp32=out_fp32)]
        if gn:
            gref, gbound = kref.group_norm64(y, gamma, beta, 1e-6, True, dtype)
            cs.append(kref.check_norm(name + " groupnorm", g, gref, gbound, dtype))
        return cs

    taps = 4 if up2x else k * k
    main = "tapgemm:conv_up2x" if up2x else ("tapgemm:conv3x3" if k == 3 else "tapgemm:linear")
    return Sub(name, call, check, main=main, ksteps=taps * -(-Cin // 64) + -(-C2 // 64), tma=tma, gn=gn, act=act,
               engines=engines)


def vt_sub(dtype, bn, B=2, Cin=72, Cout=200):
    ntok = 2 * bn + 8
    x = mk(B, ntok, Cin, dtype=dtype, seed=1)
    w = weight(Cout, Cin, 1, dtype, 2).view(Cout, Cin)
    b = mk(Cout, seed=3)
    ref = w.double() @ x.double().transpose(1, 2) + b.double()[:, None]
    mag = w.double().abs() @ x.double().abs().transpose(1, 2) + b.double().abs()[:, None]
    name = f"V^T row bias ntok={ntok} Cin={Cin}"
    return Sub(name, lambda E: (E.op_vt_proj(x, w, b), None),
               lambda y, g: [kref.check_gemm(name, y[:, :, :ntok], ref, mag, Cin, dtype)],
               main="tapgemm:vt", ksteps=-(-Cin // 64), tma=False)


def attn_sub(dtype, bn, Nq=200, heads=2, d=128):
    """The fp32 logits GEMM (Q K^T at the forced width) of the unfused attention, then softmax and P V (BN = d)."""
    Nk = 2 * bn + 8
    C = heads * d
    q, k, v = mk(1, Nq, C, dtype=dtype, seed=1), mk(1, Nk, C, dtype=dtype, seed=2), mk(1, Nk, C, dtype=dtype, seed=3)
    vt = torch.zeros(1, C, (Nk + 7) // 8 * 8, device="cuda", dtype=dtype)
    vt[:, :, :Nk] = v.transpose(1, 2)
    ref, pav, e_s, psub = kref.attention64(q, k, v, heads)
    name = f"attention logits Nq={Nq} Nk={Nk} d={d}"
    return Sub(name, lambda E: (E.op_attention(q, k, vt, heads), None),
               lambda y, g: [kref.check_attention(name, y, ref, pav, e_s, psub, Nk, dtype)],
               main="tapgemm:attn_qk", ksteps=d // 64, tma=False)


def matrix(dtype, variant, bn):
    import i2it
    tma_width = bn % 64 == 0
    n3 = 2 * bn + 64 if tma_width else 2 * bn + 8       # three n-tiles, the last one ragged (at BN = 64 only without TMA)
    c = lambda *a, **kw: conv_sub(dtype, bn, *a, **kw)
    if variant == "lean":
        every = ("default", "noostg2", "nolean")
        return [
            c("3x3 m-tiles over 4 images, 3x5 maps, Cin=72, residual", 6, 3, 5, 72, n3, res=True, engines=every),
            c("3x3 GroupNorm+SiLU partials, 12x12 maps, residual", 2, 12, 12, 64, bn + 64, res=True, gn=True, engines=every),
            c("token rows 2x150, Cin=8", 2, 1, 150, 8, n3, k=1, tokens=True, engines=every),
            c("3x3 Cin=384: 54 k-steps", 1, 8, 8, 384, bn + 64, engines=("default", "nolean")),
            c("token rows 500, 4 k-steps", 1, 1, 500, 256, n3, k=1, tokens=True, engines=("default", "noostg2")),
            c("up2x four phases, shared GroupNorm partials, x2", 2, 12, 12, 64, bn + 64, C2=72, up2x=True, gn=True, engines=every),
        ]
    subs = [
        c("3x3 m-tiles over 4 images, 3x5 maps, Cin=72, residual, quick-GELU", 6, 3, 5, 72, n3, res=True,
          act=i2it.ACT_QUICKGELU, engines=("default", "noostg2")),
        c("token rows 2x150, Cin=8, GELU", 2, 1, 150, 8, n3, k=1, tokens=True, act=i2it.ACT_GELU, engines=("default", "noostg2")),
        c("3x3 Cin=384: 54 k-steps, GELU", 1, 8, 8, 384, n3, act=i2it.ACT_GELU),
        c("token rows 500, 4 k-steps, clamp", 1, 1, 500, 256, n3, k=1, tokens=True, act=i2it.ACT_CLAMP1),
        c("GEGLU token rows 300, Cin=72", 1, 1, 300, 72, 2 * bn + (128 if tma_width else 16), k=1, tokens=True,
          act=i2it.ACT_GEGLU),
        c("3x3 fp32 out, m-tiles over 4 images, Cin=8", 6, 3, 5, 8, n3, out_fp32=True),
        c("3x3 clamp, x2, GroupNorm, 12x12 maps", 2, 12, 12, 64, 2 * bn + 32 if not tma_width else bn + 64, C2=72, gn=True,
          act=i2it.ACT_CLAMP1, engines=("default", "noostg2")),
        vt_sub(dtype, bn),
        attn_sub(dtype, bn),
        c("up2x four phases, GroupNorm, x2", 2, 12, 12, 64, bn + 64 if tma_width else 2 * bn + 32, C2=72, up2x=True, gn=True,
          engines=("nolean",)),
    ]
    if tma_width:          # the plain epilogues on the full instantiation
        subs += [c("3x3 m-tiles over 4 images, residual, no lean", 6, 3, 5, 72, n3, res=True, engines=("nolean",)),
                 c("3x3 GroupNorm+SiLU partials, residual, no lean", 2, 12, 12, 64, bn + 64, res=True, gn=True, engines=("nolean",))]
    else:
        subs += [c("3x3 m-tiles over 4 images, Cin=72, residual", 6, 3, 5, 72, n3, res=True)]
    if bn == 256:          # split-K keeps BN = 256 and takes the forced grid and ring depth
        s = c("split-K 3x3 8x8 1280->640, residual", 2, 8, 8, 1280, 640, res=True)
        s.fixed_bn, s.must, s.ksteps = 256, ("splitk_reduce",), 36
        subs.append(s)
    return subs


# ---------------------------------------------------------------------------------------------------------------------
# runs
# ---------------------------------------------------------------------------------------------------------------------
_SWITCHES = ("I2IT_NO_TMAOUT", "I2IT_NO_GNEPI", "I2IT_NO_SPLITK", "I2IT_NO_OSTG2", "I2IT_NO_LEAN", "I2IT_IDRES", "I2IT_NO_FLASH")
_ENGINE_ENV = {"default": (), "noostg2": ("I2IT_NO_OSTG2",), "nolean": ("I2IT_NO_LEAN",)}


@pytest.fixture(scope="module")
def engines():
    """Engines by (dtype, "default" | "noostg2" | "nolean"); the switches are read when an engine is created."""
    import i2it
    made = {}

    def get(dtype, kind):
        if (dtype, kind) not in made:
            saved = {k: os.environ.pop(k, None) for k in _SWITCHES}
            try:
                for k in _ENGINE_ENV[kind]:
                    os.environ[k] = "1"
                made[(dtype, kind)] = i2it.Engine(dtype, use_cuda_graph=False)
            finally:
                for k, v in saved.items():
                    os.environ.pop(k, None)
                    if v is not None:
                        os.environ[k] = v
        return made[(dtype, kind)]

    t0 = time.time()
    yield get
    print(f"\n[tapgemm matrix] module runtime {time.time() - t0:.1f} s")
    for e in made.values():
        e.close()


def execute(E, sub, bn=0, stages=0, grid=0):
    E._debug_tapgemm_override(bn, stages, grid)
    try:
        y, g = sub.call(E)
        torch.cuda.synchronize()
    finally:
        E._debug_tapgemm_override(0, 0, 0)
    ops = E.op_launches()
    return y.clone(), (g.clone() if g is not None else None), ops


def check_run(sub, kind, ops, bn, stages, grid):
    """The forced values took effect, and the main launch is the instantiation and store path this sub-case targets."""
    gemms = tapgemm_launches(ops)
    kinds = [o["kind"] for o in ops]
    where = f"{sub.name} [{kind} BN={bn} st={stages} grid={grid}]: " + "; ".join(g["kind"] + "(" + g["shape"] + ")" for g in gemms)
    mains = [g for g in gemms if g["kind"] == sub.main]
    assert mains, where
    for m in sub.must:
        assert m in kinds, where
    for g in gemms:
        if stages:
            assert g["st"] == stages, where
        if grid:
            assert g["grid"] == grid, where
        else:
            assert g["grid"] == min(g["tiles"], torch.cuda.get_device_properties(0).multi_processor_count), where
    for g in mains:
        assert g["BN"] == (sub.fixed_bn or bn), where
        tma = sub.tma if not sub.fixed_bn else False
        assert (g["mode"] != "direct") == tma, where
        if tma:
            assert (g["mode"] == "tma2") == (kind != "noostg2" and predicted_tma2(g["BN"], sub.ksteps)), where
        assert g["gn"] == (sub.gn and tma), where
        assert g["lean"] == (tma and sub.act == 0 and kind != "nolean"), where
    return where


def forced_configs(bn, ksteps, gemms, main):
    """(stages, grid) pairs beyond the engine's own: a 2-stage ring on one CTA, and a ring of (k-steps - 1) stages where the
    launch can take it (the phase flips inside a tile and carries into the next) on a grid that does not divide the n-tile
    count and leaves several tiles per CTA."""
    st0 = min(g["st"] for g in gemms)
    tiles = min(g["tiles"] for g in gemms)
    n_tiles = -(-main["N"] // main["BN"])
    out = [(2, 1)]
    grids = [g for g in (3, 5, 7, 2) if g < tiles and (n_tiles == 1 or g % n_tiles)]
    s1 = ksteps - 1 if 3 <= ksteps - 1 <= st0 else 0
    if grids:
        out.append((s1, grids[0]))
    elif s1:
        out.append((s1, 0))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("variant,bn", INSTANTIATIONS, ids=[f"{v}{n}" for v, n in INSTANTIATIONS])
@pytest.mark.parametrize("dtype", [pytest.param(bf, id="bf16"), pytest.param(hf, id="fp16")])
def test_tapgemm_instantiation(engines, dtype, variant, bn):
    t0 = time.time()
    hit, worst, mean_ulp, lines = set(), 0.0, 0.0, []
    for sub in matrix(dtype, variant, bn):
        base_y, base_g, base_ops = execute(engines(dtype, "default"), sub)     # the engine's own choices
        gn_ref = {tapgemm_launches(base_ops)[0]["gn"]: base_g}
        for kind in sub.engines:
            E = engines(dtype, kind)
            y, g, ops = execute(E, sub, bn)
            runs = [(0, 0, y, g, ops)]
            gemms = tapgemm_launches(ops)
            main = [x for x in gemms if x["kind"] == sub.main][0]
            for stages, grid in forced_configs(bn, sub.ksteps, gemms, main):
                runs.append((stages, grid) + execute(E, sub, bn, stages, grid))
            for stages, grid, y, g, ops in runs:
                where = check_run(sub, kind, ops, bn, stages, grid)
                lines.append(where)
                for c in sub.check(y, g):
                    assert c, f"{c}\n  {where}"
                    worst, mean_ulp = max(worst, c.worst), max(mean_ulp, c.mean_ulp)
                assert torch.equal(y, base_y), f"output differs from the engine's own configuration: {where}"
                if g is not None:
                    path = tapgemm_launches(ops)[0]["gn"]
                    if path in gn_ref:
                        assert torch.equal(g, gn_ref[path]), f"GroupNorm differs within its statistics path: {where}"
                    else:
                        gn_ref[path] = g
                hit |= {signature(dtype, x) for x in tapgemm_launches(ops)}
    print(f"\n[{DTYPE_NAME[dtype]} {variant} BN={bn}] worst err/bound={worst:.3f} max mean_ulp={mean_ulp:.3f} "
          f"runs={len(lines)} {time.time() - t0:.1f} s")
    for line in lines:
        print("   ", line)
    missing = declared_signatures(dtype, variant, bn) - hit
    assert not missing, f"declared signatures not exercised: {sorted(missing)}"


@pytest.mark.gpu
def test_override_rejects_illegal_values(engines):
    """A value the launch cannot take fails the op and names the legal range (a silently clamped override would test nothing);
    the next op at the engine's own choices still runs."""
    E = engines(bf, "default")
    sub = conv_sub(bf, 64, "3x3 1x8x8 64->80", 1, 8, 8, 64, 80)          # 1 m-tile x 1..5 n-tiles, 9 k-steps
    for bn, stages, grid, legal in ((200, 0, 0, "legal: 16, 32, 48, 64, 80"), (96, 0, 0, "legal: 16, 32, 48, 64, 80"),
                                    (64, 1, 0, "legal: 2..8"), (64, 9, 0, "legal: 2..8"), (64, 0, 3, "legal: 1..2"),
                                    (-1, 0, 0, ">= 0")):
        with pytest.raises(RuntimeError, match=re.escape(legal)):
            execute(E, sub, bn, stages, grid)
    y, _, ops = execute(E, sub)
    for c in sub.check(y, None):
        assert c, str(c)


# ---------------------------------------------------------------------------------------------------------------------
# production coverage
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_production_signatures_are_covered():
    """Every tapgemm signature of the BASELINE configs at SD-Turbo width (random weights, as bench.py builds them) is one the
    matrix above declares and exercises: #2 pix2pix bf16 batch 8, #4 stochastic bf16 batch 8, #5 (and #3) cyclegan fp16 a2b at
    batches 1 ... 16 on one handle."""
    import gc
    import i2it
    import weights as W
    gc.collect()                      # engines of earlier test modules still hold device memory until collected
    torch.cuda.empty_cache()
    S = 512
    seen = {}

    def collect(tag, e, dtype):
        for g in tapgemm_launches(e.profile(1)):
            seen.setdefault(signature(dtype, g), set()).add(tag)

    def engine(kind, dtype, sd):
        e = i2it.Engine(dtype, i2it.CYCLEGAN if kind == "cyclegan" else i2it.PIX2PIX, cfg=W.SD_TURBO, use_cuda_graph=False,
                        max_plans=1)
        e.load_state_dict(sd)
        adapters = ("default",) if kind == "pix2pix" else ("default_encoder", "default_decoder", "default_others")
        for a in adapters:
            e.set_adapter_scale(a, 1.0)
        e.set_adapter_scale("vae_skip", 2.0)
        return e

    def inputs(B, dtype, seed=1):
        g = torch.Generator().manual_seed(seed)
        x = (torch.rand(B, 3, S, S, generator=g) * 2 - 1).to(dtype).cuda()
        text = torch.randn(1, 77, 1024, generator=g).to(dtype).cuda()
        eps = torch.randn(B, 4, S // 8, S // 8, generator=g).to(dtype).cuda()
        return x, text, eps

    for tag, twin in (("#2", False), ("#4", True)):
        sd = W.make_state_dict("pix2pix", W.SD_TURBO, seed=0, twin=twin)
        e = engine("pix2pix", bf, sd)
        r = 0.4 if twin else 1.0
        e.finalize(r, r, r, r if twin else -1.0)
        x, text, eps = inputs(8, bf)
        noise = torch.randn_like(eps) if twin else None
        e.forward(x, text, eps, noise, r)
        torch.cuda.synchronize()
        collect(tag, e, bf)
        e.close()
        del sd
    sd = W.make_state_dict("cyclegan", W.SD_TURBO, seed=0)
    e = engine("cyclegan", hf, sd)
    e.finalize(1.0, 1.0, 1.0, -1.0)
    for B in range(1, 17):            # config #5's per-GPU sweep (#3 is its batch 16)
        x, text, eps = inputs(B, hf)
        e.forward(x, text, eps)
        torch.cuda.synchronize()
        collect("#3" if B == 16 else f"#5 b{B}", e, hf)
    e.close()
    declared = set()
    for v, n in INSTANTIATIONS:
        for dt in (bf, hf):
            declared |= declared_signatures(dt, v, n)
    print("\n[production tapgemm signatures] dtype variant BN store gn several-tiles-per-CTA | configs | in the matrix")
    for sig in sorted(seen, key=lambda s: (s[0], s[1], s[2], s[3], s[4], s[5])):
        tags = sorted(seen[sig], key=lambda t: (len(t), t))
        shown = ", ".join(tags[:6]) + (f" (+{len(tags) - 6})" if len(tags) > 6 else "")
        print(f"    {sig[0]} {sig[1]:4s} BN={sig[2]:3d} {sig[3]:6s} gn={int(sig[4])} multi={int(sig[5])} | {shown} | "
              f"{'yes' if sig in declared else 'NO'}")
    lean192 = sorted(s for s in seen if s[1] == "lean" and s[2] == 192 and "#2" in seen[s])
    print(f"    config #2 runs lean BN=192: {bool(lean192)} {lean192}")
    assert set(seen) <= declared, sorted(set(seen) - declared)


# ---------------------------------------------------------------------------------------------------------------------
# drift (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def test_matrix_lists_every_instantiation():
    """The matrix's instantiation list is TG_BN_LEAN + TG_BN_FULL of csrc/engine.cu, pick_bn's unrestricted candidates are
    TG_BN_FULL and its TMA-store candidates are lean instantiations: an instantiation added without a test fails here."""
    src = open(os.path.join(ROOT, "img2img-turbo_b200", "csrc", "engine.cu")).read()

    def macro(name):
        m = re.search(r"#define " + name + r"\(X\)(.*)", src)
        assert m, name
        return [int(v) for v in re.findall(r"X\((\d+)\)", m.group(1))]

    def cand(name):
        m = re.search(r"static const int " + name + r"\[\] = \{([^}]*)\}", src)
        assert m, name
        return [int(v) for v in re.findall(r"\d+", m.group(1))]

    lean, full = macro("TG_BN_LEAN"), macro("TG_BN_FULL")
    assert sorted(cand("cand_any")) == sorted(full)
    assert set(cand("cand_64")) <= set(lean) and set(cand("cand_128")) <= set(lean)
    assert INSTANTIATIONS == [("lean", n) for n in lean] + [("full", n) for n in full]
    assert set(SIGNATURE_MODES) == set(INSTANTIATIONS)
