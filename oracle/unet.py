"""ORACLE (test infrastructure, never imported by the product path).

Plain-PyTorch fp32 CPU restatement of the SD1.5 `UNet2DConditionModel` skeleton that the reference drives through
diffusers (third-party, absent from /root/reference: `diffusers`, recommended ==0.19.3 in README.md:66, minimum
0.18.2 in train_edlora.py:25, unpinned in requirements.txt:2).  Restated from the published diffusers-0.19.3
algorithm with runwayml/stable-diffusion-v1-5 `unet/config.json` values; anchored on the reference's call sites:
    unet(latent_model_input, t, encoder_hidden_states=prompt_embeds, cross_attention_kwargs=...).sample
        mixofshow/pipelines/pipeline_edlora.py:277-282, mixofshow/pipelines/trainer_edlora.py:237,
        gradient_fusion.py:619, mixofshow/pipelines/pipeline_regionally_t2iadapter.py:556-566
    attn.to_q/.to_k/.to_v/.to_out/.head_to_batch_dim/.get_attention_scores/...   mixofshow/models/edlora.py:64-88

Module / parameter names and the class names `Attention`, `Transformer2DModel` equal diffusers' so that the
reference's installers (edlora.py:176-218 match `layer.__class__.__name__ == 'Attention'` and `'attn2' in name`) and
its LoRA injection (trainer_edlora.py:121-133) work on this skeleton unchanged.

PARITY PINNING: the reference has no tests / golden vectors for this boundary (SURVEY.md §4, §8c) and diffusers is
not installed here, so the *skeleton* is "parity unpinned" against diffusers itself; everything the reference owns
(processors, LoRA layer, region rewrite, ...) is pinned by running the reference's own modules on this skeleton
(tests/golden/make_golden.py).
"""
import math
from types import SimpleNamespace

import torch
import torch.nn as nn
import torch.nn.functional as F

SD15 = dict(in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2,
            attention_head_dim=8, cross_attention_dim=768, norm_num_groups=32, norm_eps=1e-5)


# ------------------------------------------------------------------------------------------------ attention
class AttnProcessor:
    """diffusers' default processor (used for attn1 in the EDLoRA pipelines)."""

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None):
        if encoder_hidden_states is None:
            encoder_hidden_states = hidden_states
        query = attn.head_to_batch_dim(attn.to_q(hidden_states))
        key = attn.head_to_batch_dim(attn.to_k(encoder_hidden_states))
        value = attn.head_to_batch_dim(attn.to_v(encoder_hidden_states))
        if attn.sdpa_self and query.shape[1] == key.shape[1] and query.shape[1] > 1024:
            # mathematically identical; avoids materialising [B*8, N, N] probabilities on the CPU
            hidden_states = F.scaled_dot_product_attention(query, key, value, scale=attn.scale)
        else:
            probs = attn.get_attention_scores(query, key, attention_mask)
            hidden_states = torch.bmm(probs, value)
        hidden_states = attn.batch_to_head_dim(hidden_states)
        hidden_states = attn.to_out[0](hidden_states)
        hidden_states = attn.to_out[1](hidden_states)
        return hidden_states


class Attention(nn.Module):
    """The attribute surface the reference's processors touch (SURVEY.md §8a row U4)."""

    def __init__(self, query_dim, cross_attention_dim=None, heads=8, dim_head=64):
        super().__init__()
        inner = heads * dim_head
        cross = cross_attention_dim if cross_attention_dim is not None else query_dim
        self.heads = heads
        self.scale = dim_head ** -0.5
        self.upcast_attention = False
        self.upcast_softmax = False
        self.spatial_norm = None
        self.group_norm = None
        self.norm_cross = None
        self.residual_connection = False
        self.rescale_output_factor = 1.0
        self.sdpa_self = True
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(cross, inner, bias=False)
        self.to_v = nn.Linear(cross, inner, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(inner, query_dim), nn.Dropout(0.0)])
        self.processor = AttnProcessor()

    def set_processor(self, processor):
        self.processor = processor

    def head_to_batch_dim(self, t):
        b, n, c = t.shape
        h = self.heads
        return t.reshape(b, n, h, c // h).permute(0, 2, 1, 3).reshape(b * h, n, c // h)

    def batch_to_head_dim(self, t):
        bh, n, d = t.shape
        h = self.heads
        return t.reshape(bh // h, h, n, d).permute(0, 2, 1, 3).reshape(bh // h, n, d * h)

    def prepare_attention_mask(self, attention_mask, target_length, batch_size=None):
        assert attention_mask is None
        return None

    def get_attention_scores(self, query, key, attention_mask=None):
        dtype = query.dtype
        scores = torch.baddbmm(torch.empty(query.shape[0], query.shape[1], key.shape[1], dtype=query.dtype,
                                           device=query.device), query, key.transpose(-1, -2), beta=0,
                               alpha=self.scale)
        return scores.softmax(dim=-1).to(dtype)

    def forward(self, hidden_states, encoder_hidden_states=None, attention_mask=None, **cross_attention_kwargs):
        return self.processor(self, hidden_states, encoder_hidden_states=encoder_hidden_states,
                              attention_mask=attention_mask, **cross_attention_kwargs)


class GEGLU(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)

    def forward(self, x):
        a, g = self.proj(x).chunk(2, dim=-1)
        return a * F.gelu(g)


class FeedForward(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.net = nn.ModuleList([GEGLU(dim, dim * 4), nn.Dropout(0.0), nn.Linear(dim * 4, dim)])

    def forward(self, x):
        for m in self.net:
            x = m(x)
        return x


class BasicTransformerBlock(nn.Module):
    def __init__(self, dim, heads, dim_head, cross_attention_dim):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim)
        self.attn1 = Attention(dim, None, heads, dim_head)
        self.norm2 = nn.LayerNorm(dim)
        self.attn2 = Attention(dim, cross_attention_dim, heads, dim_head)
        self.norm3 = nn.LayerNorm(dim)
        self.ff = FeedForward(dim)

    def forward(self, x, encoder_hidden_states=None, cross_attention_kwargs=None):
        kw = cross_attention_kwargs if cross_attention_kwargs is not None else {}
        x = self.attn1(self.norm1(x), encoder_hidden_states=None, **kw) + x
        x = self.attn2(self.norm2(x), encoder_hidden_states=encoder_hidden_states, **kw) + x
        x = self.ff(self.norm3(x)) + x
        return x


class Transformer2DModel(nn.Module):
    def __init__(self, heads, dim_head, in_channels, cross_attention_dim, groups=32):
        super().__init__()
        inner = heads * dim_head
        self.norm = nn.GroupNorm(groups, in_channels, eps=1e-6, affine=True)
        self.proj_in = nn.Conv2d(in_channels, inner, 1)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(inner, heads, dim_head, cross_attention_dim)])
        self.proj_out = nn.Conv2d(inner, in_channels, 1)

    def forward(self, x, encoder_hidden_states=None, cross_attention_kwargs=None):
        b, c, h, w = x.shape
        res = x
        x = self.proj_in(self.norm(x))
        x = x.permute(0, 2, 3, 1).reshape(b, h * w, -1)
        for blk in self.transformer_blocks:
            x = blk(x, encoder_hidden_states, cross_attention_kwargs)
        x = x.reshape(b, h, w, -1).permute(0, 3, 1, 2).contiguous()
        return self.proj_out(x) + res


# ------------------------------------------------------------------------------------------------ resnet / sampling
class ResnetBlock2D(nn.Module):
    def __init__(self, in_channels, out_channels, temb_channels=1280, groups=32, eps=1e-5):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=eps)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, padding=1)
        self.time_emb_proj = nn.Linear(temb_channels, out_channels)
        self.norm2 = nn.GroupNorm(groups, out_channels, eps=eps)
        self.dropout = nn.Dropout(0.0)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, padding=1)
        self.nonlinearity = nn.SiLU()
        self.conv_shortcut = nn.Conv2d(in_channels, out_channels, 1) if in_channels != out_channels else None

    def forward(self, x, temb):
        h = self.conv1(self.nonlinearity(self.norm1(x)))
        h = h + self.time_emb_proj(self.nonlinearity(temb))[:, :, None, None]
        h = self.conv2(self.dropout(self.nonlinearity(self.norm2(h))))
        if self.conv_shortcut is not None:
            x = self.conv_shortcut(x)
        return x + h


class Downsample2D(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, stride=2, padding=1)

    def forward(self, x):
        return self.conv(x)


class Upsample2D(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, padding=1)

    def forward(self, x, output_size=None):
        if output_size is None:
            return self.conv(F.interpolate(x, scale_factor=2.0, mode='nearest'))
        return self.conv(F.interpolate(x, size=output_size, mode='nearest'))


class CrossAttnDownBlock2D(nn.Module):
    def __init__(self, cin, cout, heads, cross_dim, num_layers, add_downsample):
        super().__init__()
        self.attentions = nn.ModuleList(
            [Transformer2DModel(heads, cout // heads, cout, cross_dim) for _ in range(num_layers)])
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout) for i in range(num_layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if add_downsample else None

    def forward(self, x, temb, ehs, kw, additional_residuals=None):
        outs = ()
        n = len(self.resnets)
        for i, (resnet, attn) in enumerate(zip(self.resnets, self.attentions)):
            x = attn(resnet(x, temb), ehs, kw)
            if i == n - 1 and additional_residuals is not None:
                x = x + additional_residuals
            outs += (x,)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
            outs += (x,)
        return x, outs


class DownBlock2D(nn.Module):
    def __init__(self, cin, cout, num_layers, add_downsample):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout) for i in range(num_layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if add_downsample else None

    def forward(self, x, temb):
        outs = ()
        for resnet in self.resnets:
            x = resnet(x, temb)
            outs += (x,)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
            outs += (x,)
        return x, outs


class UNetMidBlock2DCrossAttn(nn.Module):
    def __init__(self, channels, heads, cross_dim):
        super().__init__()
        self.attentions = nn.ModuleList([Transformer2DModel(heads, channels // heads, channels, cross_dim)])
        self.resnets = nn.ModuleList([ResnetBlock2D(channels, channels), ResnetBlock2D(channels, channels)])

    def forward(self, x, temb, ehs, kw):
        x = self.resnets[0](x, temb)
        x = self.attentions[0](x, ehs, kw)
        return self.resnets[1](x, temb)


class UpBlock2D(nn.Module):
    def __init__(self, cin, prev, cout, num_layers, add_upsample):
        super().__init__()
        self.resnets = nn.ModuleList()
        for i in range(num_layers):
            skip = cin if i == num_layers - 1 else cout
            rin = prev if i == 0 else cout
            self.resnets.append(ResnetBlock2D(rin + skip, cout))
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_upsample else None

    def forward(self, x, skips, temb, upsample_size=None):
        for resnet in self.resnets:
            x = resnet(torch.cat([x, skips.pop()], dim=1), temb)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x) if upsample_size is None else self.upsamplers[0](x, upsample_size)
        return x


class CrossAttnUpBlock2D(nn.Module):
    def __init__(self, cin, prev, cout, heads, cross_dim, num_layers, add_upsample):
        super().__init__()
        self.attentions = nn.ModuleList(
            [Transformer2DModel(heads, cout // heads, cout, cross_dim) for _ in range(num_layers)])
        self.resnets = nn.ModuleList()
        for i in range(num_layers):
            skip = cin if i == num_layers - 1 else cout
            rin = prev if i == 0 else cout
            self.resnets.append(ResnetBlock2D(rin + skip, cout))
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_upsample else None

    def forward(self, x, skips, temb, ehs, kw, upsample_size=None):
        for resnet, attn in zip(self.resnets, self.attentions):
            x = attn(resnet(torch.cat([x, skips.pop()], dim=1), temb), ehs, kw)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x) if upsample_size is None else self.upsamplers[0](x, upsample_size)
        return x


def timestep_embedding(timesteps, dim=320):
    """sinusoidal embedding, flip_sin_to_cos=True, downscale_freq_shift=0 -> [cos | sin]."""
    half = dim // 2
    exponent = -math.log(10000.0) * torch.arange(half, dtype=torch.float32, device=timesteps.device) / half
    emb = timesteps[:, None].float() * torch.exp(exponent)[None, :]
    return torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1)


class TimestepEmbedding(nn.Module):
    def __init__(self, cin, dim):
        super().__init__()
        self.linear_1 = nn.Linear(cin, dim)
        self.act = nn.SiLU()
        self.linear_2 = nn.Linear(dim, dim)

    def forward(self, x):
        return self.linear_2(self.act(self.linear_1(x)))


class UNet2DConditionModel(nn.Module):
    def __init__(self, cfg=None):
        super().__init__()
        cfg = dict(SD15, **(cfg or {}))
        self.config = SimpleNamespace(sample_size=64, **cfg)
        self.in_channels = cfg['in_channels']
        ch = cfg['block_out_channels']
        heads = cfg['attention_head_dim']
        cross = cfg['cross_attention_dim']
        L = cfg['layers_per_block']
        temb_dim = ch[0] * 4
        self.conv_in = nn.Conv2d(cfg['in_channels'], ch[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(ch[0], temb_dim)
        self.down_blocks = nn.ModuleList()
        out = ch[0]
        for i, c in enumerate(ch):
            cin, out = out, c
            last = i == len(ch) - 1
            if not last:
                self.down_blocks.append(CrossAttnDownBlock2D(cin, out, heads, cross, L, True))
            else:
                self.down_blocks.append(DownBlock2D(cin, out, L, False))
        self.mid_block = UNetMidBlock2DCrossAttn(ch[-1], heads, cross)
        self.up_blocks = nn.ModuleList()
        rev = list(reversed(ch))
        out = rev[0]
        for i, c in enumerate(rev):
            prev, out = out, c
            cin = rev[min(i + 1, len(ch) - 1)]
            last = i == len(ch) - 1
            if i == 0:
                self.up_blocks.append(UpBlock2D(cin, prev, out, L + 1, True))
            else:
                self.up_blocks.append(CrossAttnUpBlock2D(cin, prev, out, heads, cross, L + 1, not last))
        self.conv_norm_out = nn.GroupNorm(cfg['norm_num_groups'], ch[0], eps=cfg['norm_eps'])
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(ch[0], cfg['out_channels'], 3, padding=1)

    def forward(self, sample, timestep, encoder_hidden_states, cross_attention_kwargs=None,
                down_block_additional_residuals=None):
        if not torch.is_tensor(timestep):
            timestep = torch.tensor([timestep], dtype=torch.long, device=sample.device)
        elif timestep.ndim == 0:
            timestep = timestep[None].to(sample.device)
        timestep = timestep.expand(sample.shape[0])
        temb = self.time_embedding(timestep_embedding(timestep, self.conv_in.out_channels).to(sample.dtype))
        is_adapter = down_block_additional_residuals is not None
        adapters = list(down_block_additional_residuals) if is_adapter else []
        x = self.conv_in(sample)
        skips = [x]
        for blk in self.down_blocks:
            if isinstance(blk, CrossAttnDownBlock2D):
                extra = adapters.pop(0) if (is_adapter and len(adapters) > 0) else None
                x, outs = blk(x, temb, encoder_hidden_states, cross_attention_kwargs, extra)
                skips += list(outs)
            else:
                x, outs = blk(x, temb)
                outs = list(outs)
                if is_adapter and len(adapters) > 0:
                    x = x + adapters.pop(0)  # diffusers does this in place: the last skip aliases x
                    outs[-1] = x
                skips += outs
        x = self.mid_block(x, temb, encoder_hidden_states, cross_attention_kwargs)
        # diffusers' forward_upsample_size: when a latent side is not a multiple of 2^(number of upsamplers), the
        # stride-2 downsamplers round up (ceil) and every non-final up block interpolates to the size of the next skip
        factor = 2 ** (len(self.up_blocks) - 1)
        forward_upsample_size = any(s % factor != 0 for s in sample.shape[-2:])
        for i, blk in enumerate(self.up_blocks):
            final = i == len(self.up_blocks) - 1
            size = None
            if forward_upsample_size and not final:
                size = skips[-len(blk.resnets) - 1].shape[2:]
            if isinstance(blk, CrossAttnUpBlock2D):
                x = blk(x, skips, temb, encoder_hidden_states, cross_attention_kwargs, size)
            else:
                x = blk(x, skips, temb, size)
        x = self.conv_out(self.conv_act(self.conv_norm_out(x)))
        return SimpleNamespace(sample=x)


def build_unet(seed=0, cfg=None):
    """Random-init SD1.5-topology UNet, default PyTorch init per layer, seeded (SURVEY.md §8d)."""
    torch.manual_seed(seed)
    return UNet2DConditionModel(cfg).eval()


TINY = dict(block_out_channels=(320, 640), layers_per_block=1)  # small variant for fast CPU tests
