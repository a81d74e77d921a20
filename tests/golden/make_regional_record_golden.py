"""Generate tests/golden/regional_record.json: the PNG name and the `.txt` configuration lines that the reference's own
`regionally_controlable_sampling.py` writes for several argument sets, so that tests/test_fused_pipeline_outputs.py pins
`image_record` without a reference checkout.  Run with MOS_REFERENCE_ROOT pointing at a checkout of
TencentARC/Mix-of-Show:
    MOS_REFERENCE_ROOT=<checkout> python tests/golden/make_regional_record_golden.py
The script runs as `__main__` in a scratch directory, in place and unmodified; the diffusers classes it loads and the
pipeline it samples with are stand-ins that return one image object, which records the path it is saved to.  Stored per
argument set: the argv, the PNG path relative to --save_dir and the text of the `.txt`.
"""
import json
import os
import runpy
import sys
import tempfile
from types import SimpleNamespace

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402

OUT = os.path.join(HERE, 'regional_record.json')

MODEL = 'experiments/composed_edlora/chilloutmix/potter+hermione+thanos_chilloutmix/combined_model_base'
NEG = 'longbody, lowres, bad anatomy, bad hands, missing fingers, extra digit, fewer digits, cropped, worst quality, low quality'
REWRITE = ('[a <potter1> <potter2>, in Hogwarts uniform, near the castle]-*-[' + NEG + ']-*-[4, 6, 1024, 490]|'
           '[a <hermione1> <hermione2>, girl, in Hogwarts uniform]-*-[' + NEG + ']-*-[14, 490, 1024, 920]|'
           '[a <thanos1> <thanos2>, purple armor]-*-[' + NEG + ']-*-[2, 1302, 1024, 1992]')
POSE, SKETCH = 'conditions/harry_hermione_thanos_2x.png', 'conditions/harry_hermione_thanos_sketch_2x.png'

CASES = {
    # no condition (the reference then has no image size, so its regions are whole-image '[]' boxes), no suffix
    'plain': ['--pretrained_model', MODEL, '--prompt', 'three people near the castle, 4K, high quality', '--negative_prompt',
              NEG, '--prompt_rewrite', '[a <potter1> <potter2>]-*-[blurry]-*-[]|[a <thanos1> <thanos2>]-*-[]-*-[]',
              '--seed', '19', '--save_dir', 'results/plain'],
    # regionally_sample.sh's real-character run: key pose only, an empty sketch condition, a suffix
    'keypose': ['--pretrained_model=' + MODEL, '--sketch_adaptor_weight=1.0', '--sketch_condition=',
                '--keypose_adaptor_weight=1.0', '--keypose_condition=' + POSE, '--save_dir=results/keypose',
                '--prompt=three people near the castle, 4K, high quality, high resolution, best quality',
                '--negative_prompt=' + NEG, '--prompt_rewrite=' + REWRITE, '--suffix=baseline', '--seed=19'],
    # both conditions with per-region adaptor weights
    'both': ['--pretrained_model', MODEL, '--keypose_condition', POSE, '--keypose_adaptor_weight', '0.8',
             '--region_keypose_adaptor_weight', '[0, 0, 1024, 490]-0.5|[14, 490, 1024, 920]-1.2',
             '--sketch_condition', SKETCH, '--sketch_adaptor_weight', '0.75',
             '--region_sketch_adaptor_weight', '[2, 1302, 1024, 1992]-0.3', '--prompt', 'a café by the sea',
             '--prompt_rewrite', REWRITE, '--seed', '7', '--suffix', 'both', '--save_dir', 'results/both'],
    # sketch only, defaults for everything else
    'sketch': ['--pretrained_model', 'fused', '--sketch_condition', SKETCH, '--save_dir', 'out', '--seed', '0'],
}


class _Image:
    saved = []

    def save(self, path, *a, **k):
        _Image.saved.append(path)


class _Pipe:
    @classmethod
    def from_pretrained(cls, *a, **k):
        return cls()

    def to(self, device):
        return self

    def set_new_concept_cfg(self, cfg):
        pass

    def __call__(self, **kw):
        return SimpleNamespace(images=[_Image()])


class _Loaded:
    @classmethod
    def from_pretrained(cls, *a, **k):
        return cls()

    def to(self, *a, **k):
        return self


def main():
    assert ref_shims.reference_available(), 'the reference checkout is needed to generate the golden data'
    from PIL import Image
    ref_shims.install_stubs()
    sys.modules['diffusers'].DPMSolverMultistepScheduler = _Loaded
    sys.modules['diffusers.models'].T2IAdapter = _Loaded
    for name in ('mixofshow', 'mixofshow.pipelines'):
        ref_shims._stub(name)
    ref_shims._stub('mixofshow.pipelines.pipeline_regionally_t2iadapter', RegionallyT2IAdapterPipeline=_Pipe)
    script = os.path.join(ref_shims.REFERENCE_ROOT, 'regionally_controlable_sampling.py')
    out, cwd, argv0 = {}, os.getcwd(), sys.argv
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            for model in (MODEL, 'fused'):
                os.makedirs(model)
                json.dump({}, open(os.path.join(model, 'new_concept_cfg.json'), 'w'))
            os.makedirs('conditions')
            Image.new('RGB', (2048, 1024)).save(POSE)
            Image.new('L', (2048, 1024)).save(SKETCH)
            for tag, argv in CASES.items():
                _Image.saved.clear()
                sys.argv = ['regionally_controlable_sampling.py'] + argv
                runpy.run_path(script, run_name='__main__')
                png, = _Image.saved
                save_dir = os.path.dirname(os.path.dirname(png))
                out[tag] = {'argv': argv, 'name': os.path.relpath(png, save_dir),
                            'txt': open(png[:-len('.png')] + '.txt', encoding='utf-8').read()}
        finally:
            os.chdir(cwd)
            sys.argv = argv0
    with open(OUT, 'w', encoding='utf-8') as f:
        json.dump(out, f, indent=1, ensure_ascii=False)
        f.write('\n')
    print(OUT, os.path.getsize(OUT))


if __name__ == '__main__':
    main()
