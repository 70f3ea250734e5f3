"""CPU: how Pix2Pix_Turbo.variations / variations_u8 find the number of variations from their arguments."""
import pytest
import torch


def _count(n=None, prompts=1, noise=None, eps=None):
    from _host import TurboBase
    t = lambda b: None if b is None else torch.zeros(b, 4, 8, 8)
    return TurboBase._variation_count(n, torch.zeros(prompts, 77, 8), t(noise), t(eps))


def test_variation_count():
    assert _count() == 1
    assert _count(n=5) == 5
    assert _count(eps=3) == 3
    assert _count(noise=4) == 4
    assert _count(prompts=2) == 2
    assert _count(n=3, prompts=3, noise=3, eps=3) == 3
    assert _count(n=3, prompts=1, noise=1) == 3          # one prompt and one noise map shared by every variation


@pytest.mark.parametrize("kw", [dict(n=2, eps=3), dict(prompts=2, noise=3), dict(n=4, prompts=3)])
def test_variation_count_disagreement(kw):
    with pytest.raises(ValueError, match="differs"):
        _count(**kw)


def test_variation_count_positive():
    with pytest.raises(ValueError, match=">= 1"):
        _count(n=0)
