"""ORACLE (test infrastructure, never imported by the product path).

Plain-PyTorch fp32 restatement of the T2I-Adapter the reference loads with
`T2IAdapter.from_pretrained('TencentARC/t2iadapter_openpose_sd14v1' / '..._sketch_sd14v1')` (regionally_controlable_sampling.py:
62-63) and calls once per image (pipeline_regionally_t2iadapter.py:474-482).  diffusers is third-party and absent here; the
network is diffusers 0.19.3 `T2IAdapter(adapter_type='full_adapter')` = `FullAdapter` [diffusers-0.19.3, from memory —
verify]:

    x = PixelUnshuffle(8)(image); x = conv_in(x)                              3x3 pad 1, Cin*64 -> channels[0]
    body[l] = AdapterBlock: AvgPool2d(2) if l > 0; in_conv (1x1) if the width changes;
              num_res_blocks x AdapterResnetBlock: x + block2(relu(block1(x)))      block1 3x3 pad 1, block2 1x1
    features = [output of body[l] for every l]

Module / parameter names equal diffusers' (`adapter.conv_in`, `adapter.body.{l}.in_conv`, `adapter.body.{l}.resnets.{k}.
block{1,2}`).  Some diffusers versions pool with ceil_mode=True; the two agree on the even sizes the GPU path accepts.
Parameter counts: 77,369,280 (Cin = 3, keypose) and 77,000,640 (Cin = 1, sketch) at channels (320, 640, 1280, 1280).
"""
from types import SimpleNamespace

import torch
import torch.nn as nn
import torch.nn.functional as F

SD_ADAPTER = dict(in_channels=3, channels=(320, 640, 1280, 1280), num_res_blocks=2, downscale_factor=8)


class AdapterResnetBlock(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.block1 = nn.Conv2d(c, c, 3, padding=1)
        self.block2 = nn.Conv2d(c, c, 1)

    def forward(self, x):
        return x + self.block2(F.relu(self.block1(x)))


class AdapterBlock(nn.Module):
    def __init__(self, cin, cout, num_res_blocks, down):
        super().__init__()
        self.down = down
        self.in_conv = nn.Conv2d(cin, cout, 1) if cin != cout else None
        self.resnets = nn.Sequential(*[AdapterResnetBlock(cout) for _ in range(num_res_blocks)])

    def forward(self, x):
        if self.down:
            x = F.avg_pool2d(x, 2)
        if self.in_conv is not None:
            x = self.in_conv(x)
        return self.resnets(x)


class FullAdapter(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        ch, n, d = cfg['channels'], cfg['num_res_blocks'], cfg['downscale_factor']
        self.d = d
        self.conv_in = nn.Conv2d(cfg['in_channels'] * d * d, ch[0], 3, padding=1)
        self.body = nn.ModuleList([AdapterBlock(ch[0], ch[0], n, False)] +
                                  [AdapterBlock(ch[i - 1], ch[i], n, True) for i in range(1, len(ch))])

    def forward(self, x):
        x = self.conv_in(F.pixel_unshuffle(x, self.d))
        feats = []
        for blk in self.body:
            x = blk(x)
            feats.append(x)
        return feats


class T2IAdapter(nn.Module):
    def __init__(self, cfg=None):
        super().__init__()
        cfg = dict(SD_ADAPTER, **(cfg or {}))
        self.config = SimpleNamespace(adapter_type='full_adapter', **{k: (list(v) if k == 'channels' else v)
                                                                     for k, v in cfg.items()})
        self.adapter = FullAdapter(cfg)

    def forward(self, x):
        return self.adapter(x)


def build_adapter(seed=0, cfg=None):
    """random-init adapter (default PyTorch init per layer), seeded"""
    torch.manual_seed(seed)
    return T2IAdapter(cfg).eval()


TINY_ADAPTER = dict(channels=(320, 640), num_res_blocks=2)   # matches oracle.unet.TINY's two down blocks
