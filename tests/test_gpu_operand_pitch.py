"""-m gpu: an operand pitch a TMA tensor map cannot express is refused while the op's plan is built.

A tensor map's strides are whole multiples of 16 bytes, so every 16-bit operand the GEMM and attention kernels load through
TMA needs a pitch that is a multiple of 8 elements.  Each case passes otherwise valid operands to a diagnostic op with one
operand's pitch 4 elements past a multiple of 8 (a column slice of a wider buffer) and expects a RuntimeError naming that
operand.  The handle stays usable: the same call with the operand at a pitch that is a multiple of 8 then gives the bits a
fresh handle gives."""
import re

import pytest
import torch

pytestmark = pytest.mark.gpu

DT = torch.bfloat16
# path: (head dim d, heads, B, Nq, Nk, kv_batch, the launch that identifies the path)
ATTN = {
    "flash_d64": (64, 2, 2, 256, 77, 1, "flash_attn"),
    "unfused_d128": (128, 2, 2, 200, 77, 1, "tapgemm:attn_qk"),
    "flash_d512": (512, 1, 1, 256, 8197, 1, "flash_attn512"),
}
ATTN_NAMES = {"q": "attention Q", "k": "attention K", "vt": "attention V^T"}


def new_engine():
    import i2it
    return i2it.Engine(DT, use_cuda_graph=False)


def ceil8(n):
    return (n + 7) // 8 * 8


def pitched(t, ld):
    """t's values as a view of a zero buffer whose last dimension has ld >= t.shape[-1] elements."""
    n = t.shape[-1]
    buf = torch.zeros(*t.shape[:-1], ld, device=t.device, dtype=t.dtype)
    buf[..., :n] = t
    return buf[..., :n]


def good(t):
    return pitched(t, ceil8(t.shape[-1]))


def bad(t):
    return pitched(t, ceil8(t.shape[-1]) + 4)


def refused(what):
    return pytest.raises(RuntimeError, match=re.escape(what) + r": pitch \d+ elements .* is not a multiple of 8")


def randn(*shape, scale=1.0, dtype=DT):
    g = torch.Generator(device="cuda").manual_seed(sum(shape))
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(dtype)


@pytest.mark.parametrize("operand", list(ATTN_NAMES))
@pytest.mark.parametrize("path", list(ATTN))
def test_attention_pitch(path, operand):
    d, heads, B, Nq, Nk, kvb, kind = ATTN[path]
    C = heads * d
    ops = {"q": randn(B, Nq, C, scale=0.5), "k": randn(kvb, Nk, C, scale=0.5), "vt": randn(kvb, C, Nk)}
    ok = {n: good(t) for n, t in ops.items()}
    E = new_engine()
    with refused(ATTN_NAMES[operand]):
        args = dict(ok, **{operand: bad(ops[operand])})
        E.op_attention(args["q"], args["k"], args["vt"], heads)
    out = E.op_attention(ok["q"], ok["k"], ok["vt"], heads)
    assert kind in [o["kind"] for o in E.op_launches()]
    ref = new_engine().op_attention(ok["q"], ok["k"], ok["vt"], heads)
    assert torch.equal(out, ref)


def test_vt_proj_pitch():
    B, ntok, Cin, Cout = 2, 77, 64, 128
    x, w, b = randn(B, ntok, Cin), randn(Cout, Cin, scale=0.1, dtype=torch.float32), randn(Cout, dtype=torch.float32)
    E = new_engine()
    with refused("vt_proj x"):
        E.op_vt_proj(bad(x), w, b)
    out = E.op_vt_proj(good(x), w, b)
    ref = new_engine().op_vt_proj(good(x), w, b)
    assert torch.equal(out[..., :ntok], ref[..., :ntok])        # columns past ntok are padding


def test_conv_x2_pitch():
    N, H, W, Cin, Cout, C2 = 1, 16, 16, 64, 64, 64
    x, x2 = randn(N, H, W, Cin), randn(N, H, W, C2)
    w, b = randn(Cout, Cin, 3, 3, scale=0.05, dtype=torch.float32), randn(Cout, scale=0.1, dtype=torch.float32)
    w2 = randn(Cout, C2, 1, 1, scale=0.1, dtype=torch.float32)
    E = new_engine()
    with refused("conv x2"):
        E.op_conv2d_ex(x, w, b, x2=bad(x2), w2=w2)
    out = E.op_conv2d_ex(x, w, b, x2=good(x2), w2=w2)
    ref = new_engine().op_conv2d_ex(x, w, b, x2=good(x2), w2=w2)
    assert torch.equal(out, ref)
