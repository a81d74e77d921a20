"""Generate tests/golden/validation_golden.pt: what the reference's own `PromptDataset` and `compose_visualize` produce in
the checks of tests/test_validation_sampling.py, so that those checks run without a reference checkout.  Run with
MOS_REFERENCE_ROOT pointing at a checkout of TencentARC/Mix-of-Show:
    MOS_REFERENCE_ROOT=<checkout> python tests/golden/make_validation_golden.py
Inputs: the two shipped test configs and their prompt files, copied under tests/golden/validation/, and a directory of
seeded synthetic PNGs that the test rebuilds.  Stored: the prompts, the (prompt, index) order and a SHA-256 of every
item's latents; the composed grid as the uint8 array the reference hands to PIL before it encodes the JPEG.
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, 'mix-of-show_b200'), os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)
from oracle import ref_shims  # noqa: E402

OUT = os.path.join(HERE, 'validation_golden.pt')


def prompt_datasets():
    import test_validation_sampling as tv
    ref = ref_shims.load_reference_module('mixofshow/data/prompt_dataset.py')
    out = {}
    for yml in tv.SHIPPED_TEST_YMLS:
        ds = ref.PromptDataset(tv.val_vis_cfg(yml))
        items = [ds[i] for i in range(len(ds))]
        out[yml] = {'prompts': list(ds.prompts), 'order': [(it['prompts'], it['indices']) for it in items],
                    'latents_sha256': [tv.sha256(it['latents']) for it in items]}
    return out


def composed_grid():
    import PIL.Image
    import test_validation_sampling as tv
    ref = ref_shims.load_reference_module('mixofshow/utils/util.py')
    captured = []

    class CaptureImage:
        """the reference's `Image` module, recording the array `compose_visualize` turns into the JPEG"""
        def __getattr__(self, k):
            return getattr(PIL.Image, k)

        def fromarray(self, a):
            captured.append(np.array(a, copy=True))
            return PIL.Image.fromarray(a)

    ref.Image = CaptureImage()
    with tempfile.TemporaryDirectory() as tmp:
        d = tv.make_compose_dir(os.path.join(tmp, 'samples'))
        ref.compose_visualize(d)
        names = sorted(f for f in os.listdir(tmp) if f.endswith('.jpg'))
    assert len(captured) == 1 and len(names) == 1
    return {'grid': torch.from_numpy(captured[0]), 'name': names[0]}


def main():
    assert ref_shims.reference_available(), 'the reference checkout is needed to generate the golden data'
    torch.save({'prompt_dataset': prompt_datasets(), 'compose': composed_grid()}, OUT)
    print(OUT, os.path.getsize(OUT))


if __name__ == '__main__':
    main()
