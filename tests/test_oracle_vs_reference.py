"""Cross-check of the oracle against the reference's own modules: what the reference computed on these seeded inputs is
stored in tests/golden/reference_live.pt (tests/golden/make_reference_live.py generates it from a reference checkout)."""
import os

import pytest
import torch

from oracle import edlora_ref as er
from oracle import inject
from oracle import unet as ou

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_live.pt')


@pytest.fixture(scope='module')
def L():
    return torch.load(GOLD, weights_only=False)


def test_reference_installer_and_lora_match_oracle(L):
    b = ou.build_unet(3, ou.TINY)
    inject.install_edlora_processors(b)
    lora = inject.random_lora_state(b, seed=4)
    inject.inject_lora(b, lora, 0.8)
    x = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(5))
    ehs = torch.randn(2, 4, 77, 768, generator=torch.Generator().manual_seed(6))
    with torch.no_grad():
        yb = b(x, torch.tensor([500, 500]), ehs).sample
    ya = L['installer_out']
    assert ((ya - yb).norm() / ya.norm()).item() < 1e-5


def test_reference_lora_target_selection_matches_trainer_rule():
    """trainer_edlora.py:121-133: every Linear/Conv2d under a module whose class name is `Attention`."""
    u = ou.build_unet(0, ou.TINY)
    names = inject.lora_target_modules(u, 'Attention')
    assert len(names) == 4 * 2 * 4  # 4 transformer blocks x (attn1, attn2) x (to_q,to_k,to_v,to_out.0)
    with torch.device('meta'):
        full = ou.UNet2DConditionModel()
    assert len(inject.lora_target_modules(full, 'Attention')) == 128


def test_reference_bind_and_quasi_newton(L):
    cfg = {'<a>': {'concept_token_names': [f'<n{i}>' for i in range(16)]}}
    assert L['bind_concept_prompt'] == er.bind_concept_prompt(['x <a> y', '<a><a>'], cfg)
    K = torch.randn(18, 32, generator=torch.Generator().manual_seed(1))
    W0 = torch.randn(24, 32, generator=torch.Generator().manual_seed(2)) * 0.1
    V = K @ (W0 + 0.05 * torch.randn(24, 32, generator=torch.Generator().manual_seed(3))).t()
    a = L['quasi_newton']
    b = er.update_quasi_newton(K, V, W0, 20)
    assert ((a - b).norm() / a.norm()).item() < 1e-5
