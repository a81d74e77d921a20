"""Drop-in for the adapter objects the reference attaches to its regional pipeline (diffusers `T2IAdapter`, loaded at
regionally_controlable_sampling.py:62-63 and called at pipeline_regionally_t2iadapter.py:474-482): `from_pretrained` of a
local diffusers-layout directory and `adapter(image) -> [feature maps]`, running on `mos_b200.adapter_engine.AdapterEngine`
(inference only).  Engines are built per input shape on first use (buffers are static).  Only adapter_type 'full_adapter'
with downscale_factor 8 (the SD1.4 / 1.5 keypose and sketch adapters) is implemented; anything else is rejected."""
from types import SimpleNamespace

import torch


class T2IAdapter:
    def __init__(self, state_dict, *, in_channels=3, channels=(320, 640, 1280, 1280), num_res_blocks=2, downscale_factor=8,
                 adapter_type='full_adapter', device='cuda'):
        from mos_b200.adapter_engine import adapter_param_shapes
        if adapter_type != 'full_adapter':
            raise ValueError(f"T2I-Adapter adapter_type={adapter_type!r} is not supported (only 'full_adapter')")
        if downscale_factor != 8:
            raise ValueError(f'T2I-Adapter downscale_factor={downscale_factor} is not supported (only 8)')
        want = adapter_param_shapes(in_channels, channels, num_res_blocks, downscale_factor)
        got = {k: tuple(v.shape) for k, v in state_dict.items()}
        if got != want:
            diff = sorted(set(got.items()) ^ set(want.items()))
            raise ValueError(f'T2I-Adapter state dict does not match its config (in_channels={in_channels}, channels='
                             f'{list(channels)}, num_res_blocks={num_res_blocks}): first differences {diff[:4]}')
        self._sd = {k: v.detach().to(torch.float32) for k, v in state_dict.items()}
        self.config = SimpleNamespace(in_channels=in_channels, channels=list(channels), num_res_blocks=num_res_blocks,
                                      downscale_factor=downscale_factor, adapter_type=adapter_type)
        self.total_downscale_factor = downscale_factor * 2 ** (len(channels) - 1)
        self.device = torch.device(device)
        self.dtype = torch.float32
        self._engines = {}

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder=None, **kw):
        """diffusers call shape (`T2IAdapter.from_pretrained(path)`, regionally_controlable_sampling.py:62-63) on a LOCAL
        directory holding config.json + diffusion_pytorch_model.safetensors (or .bin)."""
        from mixofshow.utils.model_io import load_t2i_adapter
        return load_t2i_adapter(pretrained_model_name_or_path, subfolder, **{k: v for k, v in kw.items() if k == 'device'})

    def to(self, *a, **k):
        return self

    def eval(self):
        return self

    def state_dict(self):
        return dict(self._sd)

    def parameters(self):
        return iter(self._sd.values())

    def _engine(self, B, H, W):
        from mos_b200.adapter_engine import AdapterEngine
        key = (B, H, W)
        if key not in self._engines:
            c = self.config
            self._engines[key] = AdapterEngine(self._sd, B, H, W, in_channels=c.in_channels, channels=c.channels,
                                               num_res_blocks=c.num_res_blocks, device=self.device)
        return self._engines[key]

    @torch.no_grad()
    def __call__(self, x):
        """x: [B, in_channels, H, W] image in [0, 1] -> list of fp32 NCHW feature maps [B, channels[l], H/(8 2^l), W/(8 2^l)]"""
        B, C, H, W = x.shape
        if C != self.config.in_channels:
            raise ValueError(f'T2I-Adapter expects {self.config.in_channels} input channels, got {C}')
        feats = self._engine(B, H, W).forward(x)
        out = []
        for l, (f, c) in enumerate(zip(feats, self.config.channels)):
            d = 8 * 2 ** l
            out.append(f.view(B, H // d, W // d, c).permute(0, 3, 1, 2).float().contiguous())
        return out
