"""Drop-in for the reference's `mixofshow/data/prompt_dataset.py`: the validation prompt set that `test_edlora.py` and the
validation pass of `train_edlora.py` sample (`datasets.val_vis` of every shipped config)."""
import os
import random
import re

import torch
from torch.utils.data import Dataset


class PromptDataset(Dataset):
    """`opt`: `prompts` (a prompt file path or a list of prompts), `num_samples_per_prompt`, `latent_size` (e.g.
    [4, 64, 64]), optional `replace_mapping` and `share_latent_across_prompt` (default true).

    Items are ordered sample-major: (p, i) for i in 1..num_samples_per_prompt, then p over the prompts.  Item
    {'prompts': p, 'indices': i, 'latents': randn(latent_size)}, where the latents are seeded with i, so every prompt
    of one sample index starts from the same noise."""

    def __init__(self, opt):
        self.opt = opt
        prompts = opt['prompts']
        if isinstance(prompts, list):
            pass
        elif isinstance(prompts, str) and os.path.exists(prompts):
            with open(prompts, 'r') as fr:
                prompts = [line.strip() for line in fr.readlines()]
        else:
            raise ValueError('prompts should be a prompt file path or prompt list, please check!')
        self.prompts = self.replace_placeholder(prompts)
        self.num_samples_per_prompt = opt['num_samples_per_prompt']
        self.prompts_to_generate = [(p, i) for i in range(1, self.num_samples_per_prompt + 1) for p in self.prompts]
        self.latent_size = opt['latent_size']
        self.share_latent_across_prompt = opt.get('share_latent_across_prompt', True)

    def replace_placeholder(self, prompts):
        """Applies `replace_mapping`, strips, collapses runs of spaces and drops empty lines."""
        replace_mapping = self.opt.get('replace_mapping', {}) or {}
        new_lines = []
        for line in prompts:
            if len(line.strip()) == 0:
                continue
            for k, v in replace_mapping.items():
                line = line.replace(k, v)
            line = line.strip()
            line = re.sub(' +', ' ', line)
            new_lines.append(line)
        return new_lines

    def __len__(self):
        return len(self.prompts_to_generate)

    def __getitem__(self, index):
        prompt, indice = self.prompts_to_generate[index]
        seed = indice if self.share_latent_across_prompt else random.randint(0, 1000)
        # The reference draws from torch.manual_seed(seed), which reseeds the process-global generator.  A private
        # generator with the same seed gives the same values and leaves the caller's random stream untouched.
        latents = torch.randn(self.latent_size, generator=torch.Generator().manual_seed(seed))
        return {'prompts': prompt, 'indices': indice, 'latents': latents}
