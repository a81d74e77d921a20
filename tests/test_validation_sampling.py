"""Host side of the sampling-check workflow (test_edlora.py, and the validation pass of train_edlora.py): PromptDataset
and compose_visualize against what the reference's own modules produce (tests/golden/validation_golden.pt, made by
tests/golden/make_validation_golden.py), the output names of visual_validation, the rank sharding of the prompt set,
the shipped test configs, and DPMSolverPP2M.from_pretrained."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch
import yaml
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = os.path.join(HERE, 'golden', 'validation')
GOLD = os.path.join(HERE, 'golden', 'validation_golden.pt')
SHIPPED_TEST_YMLS = ('8101_EDLoRA_potter_Cmix_B4_Repeat500.yml', '1001_EDLoRA_hina_Anyv4_B4_Iter1K.yml')

COMPOSE_PROMPTS = ('a_<new1>_<new2>_on_the_beach', 'photo_of_a_<new1>_<new2>', 'a_pencil_sketch_of_<new1>_<new2>')
COMPOSE_SAMPLES = 3
COMPOSE_HW = (24, 32)
COMPOSE_ARGS, COMPOSE_SUFFIX = 'G_7.5_S_50', 'validation_edlora_0.7'


def sha256(t):
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def val_vis_cfg(yml):
    """`datasets.val_vis` of a shipped test config, its prompt file resolved to the copy next to it"""
    with open(os.path.join(FIXTURES, yml)) as f:
        cfg = dict(yaml.safe_load(f)['datasets']['val_vis'])
    cfg['prompts'] = os.path.join(FIXTURES, os.path.basename(cfg['prompts']))
    return cfg


def make_compose_dir(path):
    """seeded random RGB PNGs named as visual_validation names them"""
    os.makedirs(path, exist_ok=True)
    g = np.random.default_rng(0)
    for prompt in COMPOSE_PROMPTS:
        for i in range(1, COMPOSE_SAMPLES + 1):
            img = g.integers(0, 256, size=(*COMPOSE_HW, 3), dtype=np.uint8)
            Image.fromarray(img).save(os.path.join(path, f'{prompt}---{COMPOSE_ARGS}---{i}---{COMPOSE_SUFFIX}.png'))
    return path


@pytest.fixture(scope='module')
def G():
    return torch.load(GOLD, weights_only=False)


# ---------------------------------------------------------------------------------------------------------- PromptDataset
@pytest.mark.parametrize('yml', SHIPPED_TEST_YMLS)
def test_prompt_dataset_matches_reference(G, yml):
    from mixofshow.data.prompt_dataset import PromptDataset
    ref = G['prompt_dataset'][yml]
    rng = torch.get_rng_state()
    ds = PromptDataset(val_vis_cfg(yml))
    items = [ds[i] for i in range(len(ds))]
    assert torch.equal(torch.get_rng_state(), rng), 'PromptDataset must not reseed the global generator'
    assert ds.prompts == ref['prompts']
    assert [(it['prompts'], it['indices']) for it in items] == [tuple(o) for o in ref['order']]
    assert [sha256(it['latents']) for it in items] == ref['latents_sha256']
    assert len(ds) == 11 * 8 and all(it['latents'].shape == (4, 64, 64) for it in items)


def test_prompt_dataset_list_and_bad_path():
    from mixofshow.data.prompt_dataset import PromptDataset
    ds = PromptDataset({'prompts': ['  a  <TOK>   dog ', '', '<TOK>'], 'num_samples_per_prompt': 2, 'latent_size': [4, 8, 8],
                        'replace_mapping': {'<TOK>': '<d1> <d2>'}})
    assert ds.prompts == ['a <d1> <d2> dog', '<d1> <d2>']
    assert [ds[i]['indices'] for i in range(len(ds))] == [1, 1, 2, 2]
    assert torch.equal(ds[0]['latents'], ds[1]['latents']) and not torch.equal(ds[0]['latents'], ds[2]['latents'])
    with pytest.raises(ValueError):
        PromptDataset({'prompts': '/nonexistent/prompts.txt', 'num_samples_per_prompt': 1, 'latent_size': [4, 8, 8]})


# ------------------------------------------------------------------------------------------------------ compose_visualize
def test_compose_visualize_matches_reference(G, tmp_path):
    from mixofshow.utils.util import GRID_PADDING, compose_grid, compose_visualize
    d = make_compose_dir(str(tmp_path / 'samples'))
    grid, name = compose_grid(d)
    ref = G['compose']['grid'].numpy()
    assert name == G['compose']['name'] == f'{COMPOSE_ARGS}---{COMPOSE_SUFFIX}.jpg'
    assert grid.shape == ref.shape and grid.dtype == np.uint8
    h, w = COMPOSE_HW
    ph, pw = h + GRID_PADDING, w + GRID_PADDING
    per_row = COMPOSE_SAMPLES + 1
    assert grid.shape[:2] == (len(COMPOSE_PROMPTS) * ph + GRID_PADDING, per_row * pw + GRID_PADDING)
    tile_mask = np.zeros(grid.shape[:2], bool)
    for r in range(len(COMPOSE_PROMPTS)):
        for c in range(per_row):
            ys, xs = slice(r * ph + GRID_PADDING, r * ph + GRID_PADDING + h), slice(c * pw + GRID_PADDING, c * pw + GRID_PADDING + w)
            tile_mask[ys, xs] = True
            if c == 0:      # prompt tile: white background in both, the text differs by font
                assert (grid[ys, xs][0, 0] == 255).all() and (ref[ys, xs][0, 0] == 255).all()
            else:
                assert np.array_equal(grid[ys, xs], ref[ys, xs]), (r, c)
    assert (grid[~tile_mask] == 0).all() and (ref[~tile_mask] == 0).all()
    compose_visualize(d)
    out = tmp_path / name
    assert out.exists() and Image.open(out).size == (grid.shape[1], grid.shape[0])


def test_compose_visualize_rejects_mixed_suffix(tmp_path):
    from mixofshow.utils.util import compose_visualize
    d = make_compose_dir(str(tmp_path / 'samples'))
    os.rename(os.path.join(d, f'{COMPOSE_PROMPTS[0]}---{COMPOSE_ARGS}---1---{COMPOSE_SUFFIX}.png'),
              os.path.join(d, f'{COMPOSE_PROMPTS[0]}---{COMPOSE_ARGS}---1---other.png'))
    with pytest.raises(AssertionError):
        compose_visualize(d)


# ------------------------------------------------------------------------------------------------------ visual_validation
class StubPipeline:
    """returns one solid-colour PIL image per prompt and records its calls"""

    def __init__(self, size=16):
        self.size, self.calls = size, []

    def __call__(self, prompt, latents, negative_prompt, num_inference_steps, guidance_scale):
        self.calls.append({'prompt': list(prompt), 'latents': latents, 'negative_prompt': negative_prompt,
                           'steps': num_inference_steps, 'guidance_scale': guidance_scale})
        return type('Out', (), {'images': [Image.new('RGB', (self.size, self.size), (10 * i, 0, 0))
                                           for i in range(len(prompt))]})()


def _val_opt(tmp_path, prompts, n, batch):
    return {'name': 'val', 'path': {'visualization': str(tmp_path / 'vis')},
            'datasets': {'val_vis': {'name': 'PromptDataset', 'prompts': prompts, 'num_samples_per_prompt': n,
                                     'latent_size': [4, 8, 8], 'replace_mapping': {'<TOK>': '<c1> <c2>'},
                                     'batch_size_per_gpu': batch}},
            'val': {'compose_visualize': True, 'alpha_list': [0, 1.0],
                    'sample': {'num_inference_steps': 50, 'guidance_scale': 7.5}}}


def test_visual_validation_names_and_batches(tmp_path):
    import test_edlora
    from mixofshow.data.prompt_dataset import PromptDataset
    from mixofshow.utils.util import NEGATIVE_PROMPT
    opt = _val_opt(tmp_path, ['photo of a <TOK>', 'a <TOK> on the beach', '<TOK>'], 2, 4)
    ds = PromptDataset(opt['datasets']['val_vis'])
    pipe = StubPipeline()
    out_dir = test_edlora.visual_validation(pipe, ds, 'validation_edlora_0.7', opt)
    assert out_dir == os.path.join(str(tmp_path / 'vis'), 'PromptDataset', 'validation_edlora_0.7')
    assert [len(c['prompt']) for c in pipe.calls] == [4, 2]                  # 6 items in batches of 4: last one short
    for c in pipe.calls:
        assert c['latents'].dtype == torch.float16 and c['latents'].shape == (len(c['prompt']), 4, 8, 8)
        assert c['negative_prompt'] == [NEGATIVE_PROMPT] * len(c['prompt'])
        assert c['steps'] == 50 and c['guidance_scale'] == 7.5
    assert torch.equal(pipe.calls[0]['latents'][0], ds[0]['latents'].half())
    expected = sorted(f'{p}---G_7.5_S_50---{i}---validation_edlora_0.7.png'
                      for p in ('photo_of_a_<c1>_<c2>', 'a_<c1>_<c2>_on_the_beach', '<c1>_<c2>') for i in (1, 2))
    assert sorted(os.listdir(out_dir)) == expected
    assert os.path.exists(os.path.join(str(tmp_path / 'vis'), 'PromptDataset', 'G_7.5_S_50---validation_edlora_0.7.jpg'))


@pytest.mark.parametrize('world', [1, 2, 3])
@pytest.mark.parametrize('n', [6, 7, 8, 12, 88])
def test_rank_shards_cover_the_set_once(world, n):
    import test_edlora
    shards = [test_edlora.rank_batches(n, 4, r, world) for r in range(world)]
    flat = [i for s in shards for b in s for i in b]
    assert sorted(flat) == list(range(n)) and len(flat) == n
    for r, s in enumerate(shards):            # rank r takes batches r, r + W, ...
        assert [b[0] // 4 for b in s] == list(range(r, -(-n // 4), world))


# ------------------------------------------------------------------------------------------------------- configs
@pytest.mark.parametrize('yml,alphas', [(SHIPPED_TEST_YMLS[0], [0, 0.7, 1.0]), (SHIPPED_TEST_YMLS[1], [0, 0.4, 0.6, 1.0])])
def test_shipped_test_configs_parse(yml, alphas):
    import test_edlora
    with open(os.path.join(FIXTURES, yml)) as f:
        opt = yaml.safe_load(f)
    assert test_edlora.alpha_list(opt) == alphas
    test_edlora.check_edlora(opt)
    assert opt['datasets']['val_vis']['batch_size_per_gpu'] == 4


def test_vanilla_lora_rejected(tmp_path):
    import test_edlora
    with open(os.path.join(FIXTURES, SHIPPED_TEST_YMLS[0])) as f:
        opt = yaml.safe_load(f)
    opt['models']['enable_edlora'] = False
    yml = tmp_path / 'lora.yml'
    yml.write_text(yaml.safe_dump(opt))
    with pytest.raises(NotImplementedError, match='enable_edlora=False'):
        test_edlora.main(['-opt', str(yml)])


# ------------------------------------------------------------------------------------------------------- scheduler
SD15_SCHEDULER_CONFIG = {'_class_name': 'PNDMScheduler', '_diffusers_version': '0.6.0', 'beta_end': 0.012,
                         'beta_schedule': 'scaled_linear', 'beta_start': 0.00085, 'num_train_timesteps': 1000,
                         'set_alpha_to_one': False, 'skip_prk_steps': True, 'steps_offset': 1, 'trained_betas': None,
                         'clip_sample': False}


def _write_scheduler(tmp_path, cfg):
    os.makedirs(tmp_path / 'scheduler', exist_ok=True)
    (tmp_path / 'scheduler' / 'scheduler_config.json').write_text(json.dumps(cfg))
    return str(tmp_path)


def _same_schedule(a, b, steps=50):
    a.set_timesteps(steps)
    b.set_timesteps(steps)
    assert np.array_equal(a.timesteps, b.timesteps)
    assert [a.coefficients(i) for i in range(steps)] == [b.coefficients(i) for i in range(steps)]


def test_scheduler_from_sd15_config(tmp_path):
    from mos_b200.scheduler import DPMSolverPP2M
    _same_schedule(DPMSolverPP2M.from_pretrained(_write_scheduler(tmp_path, SD15_SCHEDULER_CONFIG), subfolder='scheduler'),
                   DPMSolverPP2M())
    _same_schedule(DPMSolverPP2M.from_pretrained(str(tmp_path / 'missing')), DPMSolverPP2M())


def test_scheduler_config_betas_are_read(tmp_path):
    from mos_b200.scheduler import DPMSolverPP2M
    cfg = dict(SD15_SCHEDULER_CONFIG, beta_start=0.0001, beta_end=0.02, num_train_timesteps=500)
    s = DPMSolverPP2M.from_pretrained(_write_scheduler(tmp_path, cfg))
    _same_schedule(s, DPMSolverPP2M(500, 0.0001, 0.02), steps=25)
    assert s.num_train_timesteps == 500 and not np.array_equal(s.alpha_t, DPMSolverPP2M(500).alpha_t)


@pytest.mark.parametrize('key,value', [('beta_schedule', 'linear'), ('trained_betas', [0.001] * 1000),
                                       ('prediction_type', 'v_prediction'), ('solver_order', 3),
                                       ('algorithm_type', 'dpmsolver'), ('use_karras_sigmas', True),
                                       ('timestep_spacing', 'leading')])
def test_scheduler_rejects_unsupported(tmp_path, key, value):
    from mos_b200.scheduler import DPMSolverPP2M
    path = _write_scheduler(tmp_path, dict(SD15_SCHEDULER_CONFIG, **{key: value}))
    with pytest.raises(ValueError, match=key):
        DPMSolverPP2M.from_pretrained(path, subfolder='scheduler')
