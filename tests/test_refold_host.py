"""CPU: the refold entry point is exported with the right prototype, and the wrappers' choice between an in-place refold and a
new engine when a state dict changes (_host.weight_update)."""
import ctypes as C
import os
import re
import subprocess

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_refold_is_exported():
    import i2it
    hdr = open(os.path.join(ROOT, "include", "i2it.h")).read()
    for s in ("i2it_refold_weights", "i2it_debug_refold_info"):
        assert re.search(rf"\bint {s}\(", hdr), s
        assert s in i2it.SYMBOLS
    out = subprocess.run(["nm", "-D", "--defined-only", i2it.LIB_PATH], capture_output=True, text=True).stdout
    assert re.search(r"\bT i2it_refold_weights\b", out) and re.search(r"\bT i2it_debug_refold_info\b", out)


def test_refold_argtypes():
    import i2it
    lib = i2it.load_library()
    assert lib.i2it_refold_weights.argtypes == [C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float]
    assert lib.i2it_refold_weights.restype is C.c_int
    assert lib.i2it_debug_refold_info.argtypes == [C.c_void_p, C.c_char_p, C.c_size_t]
    assert lib.i2it_debug_refold_info.restype is C.c_int
    # a null handle is refused, not dereferenced
    assert lib.i2it_refold_weights(None, 1.0, 1.0, 1.0, -1.0) == 1


def _sd(twin=False):
    import weights as W
    return W.make_state_dict("pix2pix", W.TINY, seed=0, twin=twin)


def test_weight_update_decision():
    from _host import weight_record, weight_update
    sd = _sd()
    loaded = weight_record(sd)
    assert weight_update(None, sd) is None                              # no engine yet
    assert weight_update(loaded, dict(sd)) == []                        # the same tensors: nothing to register
    same_values = {k: v.clone() for k, v in sd.items()}
    assert weight_update(loaded, same_values) == []                     # equal values in new tensors
    changed = dict(sd)
    keys = [k for k in sd if ".lora_B." in k][:2] + ["vae.decoder.conv_norm_out.weight"]
    for k in keys:
        changed[k] = sd[k] + 1.0
    assert sorted(weight_update(loaded, changed)) == sorted(keys)       # in place: only what changed
    added = dict(sd)
    added["unet.extra.weight"] = torch.zeros(4)
    assert weight_update(loaded, added) is None                         # a new key
    removed = dict(sd)
    del removed[keys[0]]
    assert weight_update(loaded, removed) is None                       # a key gone
    reshaped = dict(sd)
    k = "vae.decoder.conv_norm_out.weight"
    reshaped[k] = torch.zeros(sd[k].numel() * 2)
    assert weight_update(loaded, reshaped) is None                      # a shape change
    assert weight_update(loaded, _sd(twin=True)) is None                # TwinConv added
    assert weight_update(weight_record(_sd(twin=True)), sd) is None     # TwinConv removed


def test_weight_update_sees_through_aliases():
    """The registered tensors may be the caller's own (state_dict() hands them out; an fp32 CPU tensor is stored as is):
    a tensor modified in place after registration, or handed back through an alias, is registered again."""
    from _host import weight_record, weight_update
    t, u = torch.ones(3), torch.zeros(2)
    loaded = weight_record({"a": t, "b": u})
    t.add_(1)                                                           # sd = state_dict(); sd["a"].add_(1)
    assert weight_update(loaded, {"a": t.detach().float().cpu(), "b": u}) == ["a"]
    assert weight_update(loaded, {"a": t, "b": u}) == ["a"]             # the very tensor registered, modified since
    loaded = weight_record({"a": t, "b": u})
    assert weight_update(loaded, {"a": t, "b": u}) == []
    assert weight_update(loaded, {"a": t.detach(), "b": u}) == ["a"]    # on the registered storage: no record of its values
    view = u.view(2)
    view.mul_(3)                                                        # through a view: the version counter is shared
    assert weight_update(loaded, {"a": t, "b": u}) == ["b"]
