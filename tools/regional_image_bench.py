"""Times the last step of Mix-of-Show at the size regionally_sample.sh samples (its `_2x` key-pose conditions are
2048 x 1024, W x H): one VAE decode of a 128 x 256 latent, and whole `regionally_controlable_sampling.py` runs with 3
regions, both T2I-Adapters and 50 DPM-Solver++ steps, writing the PNG.  Synthetic SD1.5-size weights: UNet, 12-layer CLIP
text encoder, VAE (tools/validation_bench.py::make_model_dir) and the two adapters (320, 640, 1280, 1280 wide).

Reports, with the card's name and power limit read in the same run:
  - ms per VAE decode of one 1024 x 2048 image (CUDA events, after a warm-up decode), and the host time of turning it
    into a PIL image and writing the PNG;
  - two CLI runs in one process after the decode measurement, wall clock to the written files; each loads and packs the
    weights again, as every run of the script does, and is split into build_model (loading), sample_image (adapters,
    engine set-up and the 50 steps), decode_latents (VAE engine set-up and the decode) and the rest (mostly the PNG
    write).  The import of torch and the first CUDA context of a fresh process are not in these times.

    python tools/regional_image_bench.py [--out DIR]
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'mix-of-show_b200'), os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'tools')):
    if p not in sys.path:
        sys.path.insert(0, p)

CONDITIONS = os.path.join(ROOT, 'tests', 'golden', 't2i_conditions')
NEG = 'longbody, lowres, bad anatomy, bad hands, missing fingers, extra digit, fewer digits, cropped, worst quality, low quality'
REGIONS = [('a <potter1> <potter2>, in Hogwarts uniform, near the castle', '[4, 6, 1024, 490]'),
           ('a <hermione1> <hermione2>, girl, in Hogwarts uniform, near the castle', '[14, 490, 1024, 920]'),
           ('a <thanos1> <thanos2>, purple armor, near the castle', '[2, 1302, 1024, 1992]')]


def make_inputs(tmp):
    """the SD1.5-size model directory, the two adapter directories and the two conditions at 2048 x 1024"""
    from PIL import Image
    from mixofshow.utils import model_io
    from oracle import adapter as oa
    from validation_bench import make_model_dir
    base = os.path.join(tmp, 'sd15')
    make_model_dir(base)
    json.dump({}, open(os.path.join(base, 'new_concept_cfg.json'), 'w'))
    argv = []
    for kind, cin, seed in (('keypose', 3, 1), ('sketch', 1, 2)):
        adapter = os.path.join(tmp, f'{kind}_adapter')
        model_io.save_t2i_adapter(oa.build_adapter(seed, dict(in_channels=cin)), adapter)
        cond = os.path.join(tmp, f'{kind}_2x.png')
        src = 'pose' if kind == 'keypose' else 'sketch'
        Image.open(os.path.join(CONDITIONS, f'harry+catA+dogA_{src}.png')).resize((2048, 1024)).save(cond)
        argv += [f'--{kind}_condition', cond, f'--{kind}_adapter', adapter]
    rewrite = '|'.join(f'[{p}]-*-[{NEG}]-*-{box}' for p, box in REGIONS)
    argv += ['--pretrained_model', base, '--prompt', 'three people near the castle, 4K, high quality', '--negative_prompt',
             NEG, '--prompt_rewrite', rewrite, '--seed', '19', '--suffix', 'baseline', '--num_inference_steps', '50']
    return base, argv


def decode_ms(base, reps):
    import torch
    from PIL import Image
    from mixofshow.pipelines.pipeline_edlora import decode_latents
    from mixofshow.utils import model_io
    from validation_bench import time_events
    vae = model_io.load_vae(base)
    z = torch.randn(1, 4, 128, 256, generator=torch.Generator().manual_seed(6)).cuda()
    vae.decode(z)
    torch.cuda.synchronize()
    ms = time_events(lambda: vae.decode(z), reps)
    with tempfile.TemporaryDirectory() as tmp:
        t = time.perf_counter()
        img = decode_latents(vae, z)[0]
        t_dec = time.perf_counter() - t
        assert isinstance(img, Image.Image) and img.size == (2048, 1024)
        t = time.perf_counter()
        img.save(os.path.join(tmp, 'x.png'))
        t_png = time.perf_counter() - t
    return {'vae_decode_ms': round(ms, 2), 'decode_latents_to_pil_s': round(t_dec, 3), 'png_write_s': round(t_png, 3)}


def cli_run(argv, save):
    """one regionally_controlable_sampling.main call, wall clock, split into its phases"""
    import torch
    import regionally_controlable_sampling as rcs
    from mixofshow.pipelines import pipeline_edlora as pe
    phases = {}
    originals = [(rcs, 'build_model'), (rcs, 'sample_image'), (pe, 'decode_latents')]
    saved = [getattr(m, n) for m, n in originals]

    def timed(name, fn):
        def run(*a, **k):
            torch.cuda.synchronize()
            t = time.perf_counter()
            out = fn(*a, **k)
            torch.cuda.synchronize()
            phases[name] = round(time.perf_counter() - t, 3)
            return out
        return run

    for (m, n), fn in zip(originals, saved):
        setattr(m, n, timed(n, fn))
    try:
        torch.cuda.synchronize()
        t = time.perf_counter()
        rcs.main(argv + ['--save_dir', save])
        torch.cuda.synchronize()
        total = time.perf_counter() - t
    finally:
        for (m, n), fn in zip(originals, saved):
            setattr(m, n, fn)
    pngs = [os.path.join(d, f) for d, _, fs in os.walk(save) for f in fs if f.endswith('.png')]
    assert len(pngs) == 1, pngs
    phases['other'] = round(total - sum(phases.values()), 3)
    return {'seconds': round(total, 2), 'phases_s': phases, 'png': os.path.relpath(pngs[0], save)}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='directory for the JSON result (default: print only)')
    ap.add_argument('--decode-reps', type=int, default=5)
    args = ap.parse_args(argv)
    import torch
    from validation_bench import card
    assert torch.cuda.is_available(), 'regional_image_bench needs a GPU'
    result = {'card': card(), 'size': '1024x2048', 'regions': 3, 'adapters': ['keypose', 'sketch'], 'steps': 50}
    with tempfile.TemporaryDirectory() as tmp:
        t = time.perf_counter()
        base, cli = make_inputs(tmp)
        result['setup_s'] = round(time.perf_counter() - t, 1)
        result.update(decode_ms(base, args.decode_reps))
        torch.cuda.empty_cache()
        result['cli_runs'] = [cli_run(cli, os.path.join(tmp, f'run{i}')) for i in range(2)]
        result['peak_allocated_gb'] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 1)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'regional_image_bench.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
