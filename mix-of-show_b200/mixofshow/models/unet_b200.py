"""GPU `UNet2DConditionModel`: the object the reference's entry points call as
`unet(sample, t, encoder_hidden_states=..., cross_attention_kwargs=..., down_block_additional_residuals=...).sample`
(mixofshow/pipelines/pipeline_edlora.py:277, trainer_edlora.py:237, gradient_fusion.py:619,
pipeline_regionally_t2iadapter.py:556).

It is an nn.Module *container*: parameters live in diffusers-named sub-modules (`down_blocks.0.attentions.0.
transformer_blocks.0.attn2.to_q`, ...; class names `Attention` / `Transformer2DModel` as diffusers) so that the
reference's `named_modules()`-driven LoRA injection (trainer_edlora.py:121-133), its processor installers
(edlora.py:176-218) and its checkpoint key mapping (convert_edlora_to_diffusers.py:43-50) work unchanged.
`forward` never executes those sub-modules: it packs their weights (plus any LoRALinearLayer / processor descriptors
found on them) into a `mos_b200.engine.UNetEngine` and runs the captured CUDA step.  No torch arithmetic fallback.
"""
from types import SimpleNamespace

import torch
import torch.nn as nn

from mos_b200.engine import UNetEngine, ehs_to_layer_major

SD15 = dict(in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2,
            attention_head_dim=8, cross_attention_dim=768, norm_num_groups=32, sample_size=64)


def _no_forward(self, *a, **k):
    raise RuntimeError(f'{self.__class__.__name__}.forward is not executed on the GPU path: call the UNet '
                       '(whole-step engine) or an attention processor (operator level) instead')


class Attention(nn.Module):
    """Parameter holder + the attribute surface the processors read (SURVEY.md §8a row U4)."""

    def __init__(self, query_dim, cross_attention_dim=None, heads=8, dim_head=64):
        super().__init__()
        inner = heads * dim_head
        cross = cross_attention_dim if cross_attention_dim is not None else query_dim
        self.heads, self.scale = heads, dim_head ** -0.5
        self.upcast_attention = self.upcast_softmax = False
        self.spatial_norm = self.group_norm = self.norm_cross = None
        self.residual_connection, self.rescale_output_factor = False, 1.0
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(cross, inner, bias=False)
        self.to_v = nn.Linear(cross, inner, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(inner, query_dim), nn.Dropout(0.0)])
        from mixofshow.models.edlora import AttnProcessor
        self.processor = AttnProcessor()

    def set_processor(self, processor):
        self.processor = processor

    def prepare_attention_mask(self, attention_mask, target_length, batch_size=None):
        assert attention_mask is None
        return None

    def forward(self, hidden_states, encoder_hidden_states=None, attention_mask=None, **cross_attention_kwargs):
        return self.processor(self, hidden_states, encoder_hidden_states=encoder_hidden_states,
                              attention_mask=attention_mask, **cross_attention_kwargs)


class GEGLU(nn.Module):
    forward = _no_forward

    def __init__(self, d_in, d_out):
        super().__init__()
        self.proj = nn.Linear(d_in, d_out * 2)


class FeedForward(nn.Module):
    forward = _no_forward

    def __init__(self, dim):
        super().__init__()
        self.net = nn.ModuleList([GEGLU(dim, dim * 4), nn.Dropout(0.0), nn.Linear(dim * 4, dim)])


class BasicTransformerBlock(nn.Module):
    forward = _no_forward

    def __init__(self, dim, heads, dim_head, cross_dim):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim)
        self.attn1 = Attention(dim, None, heads, dim_head)
        self.norm2 = nn.LayerNorm(dim)
        self.attn2 = Attention(dim, cross_dim, heads, dim_head)
        self.norm3 = nn.LayerNorm(dim)
        self.ff = FeedForward(dim)


class Transformer2DModel(nn.Module):
    forward = _no_forward

    def __init__(self, heads, dim_head, channels, cross_dim):
        super().__init__()
        self.norm = nn.GroupNorm(32, channels, eps=1e-6)
        self.proj_in = nn.Conv2d(channels, heads * dim_head, 1)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(heads * dim_head, heads, dim_head, cross_dim)])
        self.proj_out = nn.Conv2d(heads * dim_head, channels, 1)


class ResnetBlock2D(nn.Module):
    forward = _no_forward

    def __init__(self, cin, cout, temb=1280):
        super().__init__()
        self.norm1 = nn.GroupNorm(32, cin, eps=1e-5)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.time_emb_proj = nn.Linear(temb, cout)
        self.norm2 = nn.GroupNorm(32, cout, eps=1e-5)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        if cin != cout:
            self.conv_shortcut = nn.Conv2d(cin, cout, 1)


class _Resample(nn.Module):
    forward = _no_forward

    def __init__(self, c, stride):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride=stride, padding=1)


class _Block(nn.Module):
    forward = _no_forward


class TimestepEmbedding(nn.Module):
    forward = _no_forward

    def __init__(self, cin, dim):
        super().__init__()
        self.linear_1 = nn.Linear(cin, dim)
        self.linear_2 = nn.Linear(dim, dim)


class UNet2DConditionModel(nn.Module):
    def __init__(self, **cfg):
        super().__init__()
        cfg = dict(SD15, **cfg)
        self.config = SimpleNamespace(**cfg)
        self.in_channels = cfg['in_channels']
        ch, L = tuple(cfg['block_out_channels']), cfg['layers_per_block']
        heads, cross = cfg['attention_head_dim'], cfg['cross_attention_dim']
        nb = len(ch)
        self.conv_in = nn.Conv2d(cfg['in_channels'], ch[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(ch[0], 4 * ch[0])
        self.down_blocks = nn.ModuleList()
        out = ch[0]
        for i, c in enumerate(ch):
            cin, out = out, c
            blk = _Block()
            if i < nb - 1:
                blk.attentions = nn.ModuleList([Transformer2DModel(heads, c // heads, c, cross) for _ in range(L)])
            blk.resnets = nn.ModuleList([ResnetBlock2D(cin if j == 0 else c, c, 4 * ch[0]) for j in range(L)])
            if i < nb - 1:
                blk.downsamplers = nn.ModuleList([_Resample(c, 2)])
            self.down_blocks.append(blk)
        mid = _Block()
        mid.attentions = nn.ModuleList([Transformer2DModel(heads, ch[-1] // heads, ch[-1], cross)])
        mid.resnets = nn.ModuleList([ResnetBlock2D(ch[-1], ch[-1], 4 * ch[0]) for _ in range(2)])
        self.mid_block = mid
        self.up_blocks = nn.ModuleList()
        rev = list(reversed(ch))
        out = rev[0]
        for i, c in enumerate(rev):
            prev, out = out, c
            cin = rev[min(i + 1, nb - 1)]
            blk = _Block()
            if i > 0:
                blk.attentions = nn.ModuleList([Transformer2DModel(heads, c // heads, c, cross) for _ in range(L + 1)])
            blk.resnets = nn.ModuleList()
            for j in range(L + 1):
                skip = cin if j == L else c
                rin = prev if j == 0 else c
                blk.resnets.append(ResnetBlock2D(rin + skip, c, 4 * ch[0]))
            if i < nb - 1:
                blk.upsamplers = nn.ModuleList([_Resample(c, 1)])
            self.up_blocks.append(blk)
        self.conv_norm_out = nn.GroupNorm(32, ch[0], eps=1e-5)
        self.conv_out = nn.Conv2d(ch[0], cfg['out_channels'], 3, padding=1)
        self._engines = {}
        self._checked = None
        self.merge_lora = False
        self.use_graph = True
        self.act_dtype = torch.float16      # operand type of the engine (fp16 = the reference's sampling precision)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder='unet', **unused):
        """diffusers call shape (`UNet2DConditionModel.from_pretrained(path, subfolder='unet')`, trainer_edlora.py:44):
        loads a diffusers-layout directory (mixofshow/utils/model_io.py)."""
        from mixofshow.utils.model_io import load_unet
        return load_unet(pretrained_model_name_or_path, subfolder)

    def save_pretrained(self, save_directory, **unused):
        from mixofshow.utils.model_io import save_unet
        save_unet(self, save_directory, subfolder=None)

    def invalidate(self):
        """Force a re-pack on the next call (needed only after edits that bypass autograd's version counters, e.g.
        writes through `.data` such as the reference's `param.data.copy_`; optimiser steps, `load_state_dict`, `.to()`
        and LoRA / processor installation are detected)."""
        self._engines = {}
        self._checked = None

    def _load_from_state_dict(self, *a, **k):
        self._checked = None
        return super()._load_from_state_dict(*a, **k)

    def _apply(self, fn, *a, **k):
        self._checked = None
        self._engines = {}
        return super()._apply(fn, *a, **k)

    # ------------------------------------------------------------------------------------------ descriptors
    def _fingerprint(self):
        """Version walk over the parameters and LoRA descriptors.  Host-only: tensor version counters and pointers, no
        device read (alpha is tracked through its version counter; its VALUE is read once, when packing)."""
        fp = 0
        for p in self.parameters():
            fp = (fp * 1000003 + p._version + (p.data_ptr() & 0xFFFF)) & 0xFFFFFFFFFFFF
        for m in self.modules():
            l = getattr(m, '_mos_lora', None)
            if l is not None:
                fp = (fp * 1000003 + l.lora_down.weight._version + l.lora_up.weight._version * 7
                      + l.alpha._version * 13 + (l.lora_up.weight.data_ptr() & 0xFFFF)) & 0xFFFFFFFFFFFF
            if m.__class__.__name__ == 'Attention':
                fp = (fp * 1000003 + (id(m.processor) & 0xFFFFFF)) & 0xFFFFFFFFFFFF
        return fp

    def _collect_lora(self):
        lora, alpha = {}, None
        for name, m in self.named_modules():
            l = getattr(m, '_mos_lora', None)
            if l is not None:
                lora[name + '.lora_down.weight'] = l.lora_down.weight
                lora[name + '.lora_up.weight'] = l.lora_up.weight
                a = float(l.alpha)
                if alpha is not None and abs(alpha - a) > 1e-12:
                    raise ValueError('all LoRA layers of one UNet must share alpha on the fused path')
                alpha = a
        return (lora or None), (1.0 if alpha is None else alpha)

    def _collect_processors(self):
        """Returns (kind, controller): verifies that the installed cross_attention_idx equals the DFS order."""
        kinds, controller, idx = set(), None, []
        for name, m in self.named_modules():
            if m.__class__.__name__ == 'Attention' and name.endswith('attn2'):
                p = m.processor
                kinds.add(p.__class__.__name__)
                idx.append(getattr(p, 'cross_attention_idx', None))
                controller = getattr(p, 'controller', controller)
        if any(i is not None for i in idx) and idx != list(range(len(idx))):
            raise ValueError(f'cross_attention_idx assignment {idx} does not follow the reference order')
        if len(kinds) > 1:
            raise ValueError(f'mixed attention processors {kinds} are not supported')
        return (kinds.pop() if kinds else 'AttnProcessor'), controller

    def _state(self):
        """(fingerprint, processor kind, controller) of the container, re-derived by walking the module tree.  The walk
        costs ~3 ms of host time, so a denoise loop does it ONCE (`session()`), not once per step."""
        fp = self._fingerprint()
        kind, controller = self._collect_processors()
        self._checked = (fp, kind, controller)
        return self._checked

    def _engine(self, B, H, W, device, emit_probs, fp):
        key = (B, H, W, str(device), emit_probs, self.act_dtype)
        ent = self._engines.get(key)
        if ent is None or ent[0] != fp:
            lora, alpha = self._collect_lora()
            c = self.config
            eng = UNetEngine(self.state_dict(), B, H, W, lora=lora, lora_alpha=alpha, merge_lora=self.merge_lora,
                             device=device, block_out=tuple(c.block_out_channels), layers=c.layers_per_block,
                             heads=c.attention_head_dim, cross_dim=c.cross_attention_dim, emit_probs=emit_probs,
                             use_graph=self.use_graph, act_dtype=self.act_dtype)
            self._engines = {k: v for k, v in self._engines.items() if v[0] == fp}
            self._engines[key] = ent = (fp, eng)
        return ent[1]

    # ------------------------------------------------------------------------------------------ forward
    @torch.no_grad()
    def session(self, batch, height, width, device, encoder_hidden_states, cross_attention_kwargs=None,
                down_block_additional_residuals=None):
        """Prepare a denoise loop: verify / pack the weights once, upload the step-invariant inputs (layer-wise text
        embeddings, region embeddings and boxes, adapter residuals) once, and return a `DenoiseSession` whose `step()`
        is one CUDA-graph replay with no host-side tree walk, no host<->device synchronisation and no per-step copies.
        `EDLoRAPipeline.__call__` / `RegionallyT2IAdapterPipeline.__call__` drive their loops through this;
        `forward()` (the reference's `unet(...)` call shape) is `session(...)` + one step."""
        device = torch.device(device)
        fp, kind, controller = self._state()
        emit = kind == 'EDLoRA_Control_AttnProcessor' and controller is not None \
            and controller.__class__.__name__ != 'DummyController'
        eng = self._engine(batch, height, width, device, emit, fp)
        nx = len(eng.xattn_names)
        ehs = encoder_hidden_states
        if ehs.ndim == 4 and kind == 'AttnProcessor':
            raise ValueError('layer-wise (4-D) embeddings need the ED-LoRA processors '
                             '(revise_edlora_unet_attention_forward)')
        kw = cross_attention_kwargs or {}
        if kind == 'RegionT2I_AttnProcessor':
            regs = [(ehs_to_layer_major(emb.to(device), nx, eng.ACT), box) for emb, box in kw['region_list']]
            eng.set_regions(regs, (kw['height'], kw['width']))
        else:
            eng.set_regions(None, None)
        if down_block_additional_residuals is not None:
            eng.set_adapters([a.to(device).permute(0, 2, 3, 1).reshape(-1, a.shape[1]).to(eng.ACT)
                              for a in down_block_additional_residuals])
        else:
            eng.set_adapters(None)
        eng.use_graph = self.use_graph
        eng.in_ehs.copy_(ehs_to_layer_major(ehs.to(device), nx, eng.ACT), non_blocking=True)
        return DenoiseSession(self, eng, controller if emit else None)

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, cross_attention_kwargs=None,
                down_block_additional_residuals=None, return_dict=True):
        if not sample.is_cuda:
            raise RuntimeError('the GPU UNet needs CUDA tensors (there is no CPU fallback)')
        B, _, H, W = sample.shape
        sess = self.session(B, H, W, sample.device, encoder_hidden_states, cross_attention_kwargs,
                            down_block_additional_residuals)
        if not torch.is_tensor(timestep):
            timestep = torch.tensor([float(timestep)], device=sample.device)
        sess.eng.in_latents.copy_(sample)
        sess.eng.in_t.copy_(timestep.to(sample.device, torch.float32).reshape(-1).expand(B))
        out = sess.step().to(sample.dtype).clone()
        return SimpleNamespace(sample=out) if return_dict else (out,)

    def _feed_controller(self, eng, controller):
        """Hand the 16 probability maps to the controller in layer order, with the reference's call protocol
        (`controller(probs, is_cross, place)`, mixofshow/utils/ptp_util.py:37-53)."""
        nb = len(eng.block_out)
        n_down = (nb - 1) * eng.layers
        for i in range(len(eng.xattn_names)):
            place = 'down' if i < n_down else ('mid' if i == n_down else 'up')
            key = [k for k in eng.bufs if k[0] == f'probs{i}'][0]
            controller(eng.bufs[key].clone(), True, place)


class DenoiseSession:
    """One prepared denoise loop on the engine (see `UNet2DConditionModel.session`).  `latents_in` / `t_in` are the
    engine's static input buffers (fp32 NCHW [B,4,H,W] and [B]): the fused CFG + DPM-Solver++ kernel writes the next
    step's UNet input and timestep straight into them.  `step()` returns the engine's static eps buffer (NOT a copy)."""

    def __init__(self, unet, eng, controller):
        self.unet, self.eng, self.controller = unet, eng, controller
        self.latents_in, self.t_in = eng.in_latents, eng.in_t

    def step(self):
        self.eng.run()
        if self.controller is not None:
            self.unet._feed_controller(self.eng, self.controller)
        return self.eng.out_eps
