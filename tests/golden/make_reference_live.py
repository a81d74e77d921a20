"""Generate tests/golden/reference_live.pt: what the reference's own modules compute in the checks of
tests/test_oracle_vs_reference.py and tests/test_checkpoint_formats.py, so that those checks run without a reference
checkout.  Run with MOS_REFERENCE_ROOT pointing at a checkout of TencentARC/Mix-of-Show:
    MOS_REFERENCE_ROOT=<checkout> python tests/golden/make_reference_live.py
The inputs are rebuilt from the same seeds by the tests; only the reference's outputs are stored (merged weights as a
seeded sample of each changed tensor, so that the file stays small).
"""
import os
import sys
from types import SimpleNamespace

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, 'mix-of-show_b200'), os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)
from oracle import inject, ref_shims  # noqa: E402
from oracle import unet as ou  # noqa: E402

OUT = os.path.join(HERE, 'reference_live.pt')
MERGE_SAMPLE = 256          # values stored per changed weight tensor


def installer_output():
    """tests/test_oracle_vs_reference.py::test_reference_installer_and_lora_match_oracle: the reference's
    revise_edlora_unet_attention_forward + LoRALinearLayer on the tiny oracle UNet."""
    ed = ref_shims.load_reference_module('mixofshow/models/edlora.py')
    a = ou.build_unet(3, ou.TINY)
    ed.revise_edlora_unet_attention_forward(a)
    lora = inject.random_lora_state(a, seed=4)
    mods = dict(a.named_modules())
    keep = []
    for k in lora:
        if k.endswith('.lora_down.weight'):
            n = k[:-len('.lora_down.weight')]
            layer = ed.LoRALinearLayer(n, mods[n], rank=4, alpha=0.8)
            layer.lora_down.weight.data = lora[k].clone()
            layer.lora_up.weight.data = lora[n + '.lora_up.weight'].clone()
            keep.append(layer)
    x = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(5))
    ehs = torch.randn(2, 4, 77, 768, generator=torch.Generator().manual_seed(6))
    with torch.no_grad():
        return a(x, torch.tensor([500, 500]), ehs).sample


def bind_and_quasi_newton():
    pe = ref_shims.load_reference_module('mixofshow/pipelines/pipeline_edlora.py')
    gf = ref_shims.load_reference_module('gradient_fusion.py')
    cfg = {'<a>': {'concept_token_names': [f'<n{i}>' for i in range(16)]}}
    bind = pe.bind_concept_prompt(['x <a> y', '<a><a>'], cfg)
    K = torch.randn(18, 32, generator=torch.Generator().manual_seed(1))
    W0 = torch.randn(24, 32, generator=torch.Generator().manual_seed(2)) * 0.1
    V = K @ (W0 + 0.05 * torch.randn(24, 32, generator=torch.Generator().manual_seed(3))).t()
    return bind, gf.update_quasi_newton(K, V, W0.clone(), 20, 'cpu')


def checkpoint_mirror():
    """tests/test_checkpoint_formats.py::test_mirror_matches_reference_file: the reference's merge_lora_into_weight and
    load_new_concept."""
    import test_checkpoint_formats as tc
    from transformers import CLIPTextConfig, CLIPTextModel
    ref = ref_shims.load_reference_module('mixofshow/utils/convert_edlora_to_diffusers.py')
    unet = ou.build_unet(0, ou.TINY)
    clip, clip_sd = tc._clip_sd()
    ckpt = tc._delta(unet, clip, seed=5)['params']
    merge = {}
    for model_type, sd in (('unet', unet.state_dict()), ('text_encoder', clip_sd)):
        a = ref.merge_lora_into_weight(sd, ckpt[model_type], model_type=model_type, alpha=0.7)
        changed = sorted(k for k in a if not torch.equal(a[k], sd[k]))
        samples = {}
        for i, k in enumerate(changed):
            flat = a[k].reshape(-1)
            idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(i))[:MERGE_SAMPLE].clone()
            samples[k] = (idx, flat[idx].clone())
        merge[model_type] = {'keys': sorted(a.keys()), 'changed': changed, 'samples': samples}
    torch.manual_seed(0)
    m = CLIPTextModel(CLIPTextConfig(vocab_size=300, hidden_size=768, intermediate_size=3072, num_hidden_layers=1,
                                     num_attention_heads=12, max_position_embeddings=77))
    pipe = SimpleNamespace(tokenizer=tc.FakeTokenizer(300), text_encoder=m)
    pipe, cfg = ref.load_new_concept(pipe, ckpt['new_concept_embedding'], True)
    return merge, {'cfg': cfg, 'rows': m.get_input_embeddings().weight.data[300:].clone()}


def main():
    assert ref_shims.reference_available(), 'the reference checkout is needed to generate the golden data'
    bind, qn = bind_and_quasi_newton()
    merge, concept = checkpoint_mirror()
    torch.save({'installer_out': installer_output(), 'bind_concept_prompt': bind, 'quasi_newton': qn,
                'merge_lora': merge, 'load_new_concept': concept}, OUT)
    print(OUT, os.path.getsize(OUT))


if __name__ == '__main__':
    main()
