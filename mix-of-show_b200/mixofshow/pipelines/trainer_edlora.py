"""GPU mirror of the reference trainer (mixofshow/pipelines/trainer_edlora.py:20-380).

`EDLoRATrainer` keeps the reference's constructor (`EDLoRATrainer(**opt['models'])`, train_edlora.py:50), its public names
(`init_new_concept`, `set_finetune_cfg`, `get_params_to_optimize`, `get_all_concept_token_ids`, `forward`,
`delta_state_dict`, `load_delta_state_dict`) and its checkpoint layout ({'new_concept_embedding', 'text_encoder', 'unet'},
keys f'{module}.lora_down.weight' / '.lora_up.weight', :371-378), and trains any non-empty subset of the THREE parameter
groups of :82-139 — the new-concept embedding rows, the text-encoder LoRA and the UNet LoRA — in one captured CUDA graph:
text encoder forward -> UNet forward -> masked MSE + attention regulariser -> UNet backward -> text encoder backward
(mos_b200/train_engine.py + mos_b200/clip_train_engine.py).  A frozen group costs nothing: a UNet without LoRA runs plain
GEMMs and no LoRA-gradient launch; a frozen text encoder without trained rows runs its forward only (no d(text
embeddings), no CLIP backward); untrained concept rows are constants of the text encoder's token table.  The gradients land in ONE flat fp32 buffer (the payload of the
step's single NCCL all-reduce); there is no autograd graph to call `.backward()` on.  `forward` takes images (encoded by
the GPU VAE engine, :203-204) or already encoded latents.

`UNetLoRATrainer` is the latents-and-embeddings level trainer of the UNet LoRA group alone (text encoder frozen and run
upstream).

LoRA placement (`lora_cfg.where`, trainer_edlora.py:100-133): the UNet takes `Attention` or `Transformer2DModel`, the text
encoder `CLIPAttention` or `CLIPEncoderLayer`, in any combination.

Vanilla LoRA (`enable_edlora: false`, trainer_edlora.py:156-160, :220-234): one token `<new{k}>` and one embedding row per
concept word, prompts tokenized as written (no `bind_concept_prompt`), one text-encoder pass per sample, and the one
[b, 77, 768] embedding shared by all 16 cross-attention layers (TrainEngine(shared_ehs=True)).  A concept row only receives
a gradient when a prompt contains its `<new{k}>` token literally: a `replace_mapping` such as `<TOK>: <potter1> <potter2>`
does not produce those tokens, so with it the rows stay where they were initialised, as in the reference."""
import math
import re

import torch

from mos_b200.clip_train_engine import CLIP_WHERE
from mos_b200.engine import ehs_to_layer_major
from mos_b200.train_engine import UNET_WHERE, TrainEngine

VANILLA_LORA_UNSUPPORTED = ('enable_edlora=False (vanilla LoRA) checkpoints cannot be sampled by EDLoRAPipeline, so neither '
                            'test_edlora.py nor val.val_during_save takes them (the reference fails there too): sample '
                            'a lora_model-*.pth with StableDiffusionPipeline.from_pretrained(...) and '
                            'convert_edlora(pipe, ckpt, enable_edlora=False, alpha=...)')


FINETUNE_GROUPS = ('text_embedding', 'text_encoder', 'unet')


def _n_layers(text_state_dict):
    return 1 + max(int(k.split('.layers.')[1].split('.')[0]) for k in text_state_dict if '.layers.' in k)


def _check_rank(lora_cfg):
    rank = int(lora_cfg.get('rank', 4))
    if not 1 <= rank <= 4:
        raise ValueError('LoRA rank must be in 1..4 (fused epilogue)')
    return rank, float(lora_cfg.get('alpha', 1.0))


def check_lora_ranks(lora, rank, part):
    """Refuses (ValueError) a LoRA state dict of `part` ('unet' / 'text_encoder') whose rank is not the configured `rank`:
    every lora_down [r, K] (or [r, K, 1, 1]) and lora_up [N, r] (or [N, r, 1, 1]) must have r == rank, and a module's down
    and up must agree.  The flat training state keeps four rank slots per module whatever the rank, so a mismatch would
    otherwise load without error: a rank-4 checkpoint under `rank: 2` trains four ranks and saves two, a rank-2 checkpoint
    under `rank: 4` trains two and saves two zero rows.  The reference raises here too: it copies each tensor into a
    parameter of the configured shape (trainer_edlora.py:335-340)."""
    modules = dict.fromkeys(k.rsplit('.lora_', 1)[0] for k in lora if k.endswith(('.lora_down.weight', '.lora_up.weight')))
    for m in modules:
        d, u = lora.get(m + '.lora_down.weight'), lora.get(m + '.lora_up.weight')
        ranks = {r for r in (d.shape[0] if d is not None else None, u.shape[1] if u is not None else None) if r is not None}
        if ranks != {rank}:
            shapes = ', '.join(f'lora_{s} {tuple(t.shape)}' for s, t in (('down', d), ('up', u)) if t is not None)
            why = 'down and up disagree on the rank' if len(ranks) > 1 else f'rank {ranks.pop()}'
            raise ValueError(f'{part} LoRA of {m}: {shapes}: {why}, the config trains rank {rank}')


def _check_where(where, allowed, part):
    if where not in allowed:
        raise NotImplementedError(f"{part} lora_cfg.where: {where!r} is not one of the reference's placements {allowed}")
    return where


class UNetLoRATrainer:
    def __init__(self, unet_state_dict, batch_size_per_gpu, new_concept_cfg=None, finetune_cfg=None, noise_offset=None,
                 attn_reg_weight=None, reg_full_identity=True, use_mask_loss=True, latent_size=(64, 64),
                 unet_topology=None, device='cuda', seed=0, lora_state=None):
        if finetune_cfg is None:
            raise ValueError('finetune_cfg is required (trainer_edlora.py:66-67)')
        self.new_concept_cfg = dict(new_concept_cfg or {})
        self.noise_offset = noise_offset
        self.attn_reg_weight = attn_reg_weight
        self.reg_full_identity = reg_full_identity
        self.use_mask_loss = use_mask_loss
        self.device = torch.device(device)
        self.batch = int(batch_size_per_gpu)
        self.latent_size = tuple(latent_size)
        self._topo = dict(unet_topology or {})
        self._gen = torch.Generator(device='cpu').manual_seed(seed)
        self._sd = unet_state_dict
        self.set_finetune_cfg(finetune_cfg, lora_state)

    # ------------------------------------------------------------------------------------------ configuration
    def set_finetune_cfg(self, finetune_cfg, lora_state=None):
        """trainer_edlora.py:71-142.  Only the `unet` group exists on this path."""
        for part in ('text_embedding', 'text_encoder'):
            if finetune_cfg.get(part, {}).get('enable_tuning'):
                raise NotImplementedError(f"finetune_cfg['{part}'].enable_tuning: the CLIP side of ED-LoRA training is "
                                          'not built on the GPU path yet (SURVEY.md §8f); disable it')
        ucfg = finetune_cfg['unet']
        if not (ucfg.get('enable_tuning') and ucfg.get('lora_cfg')):
            raise ValueError("finetune_cfg['unet'] must enable tuning with a lora_cfg")
        lora_cfg = dict(ucfg['lora_cfg'])
        self.where = _check_where(lora_cfg.pop('where'), UNET_WHERE, 'unet')
        self.rank = int(lora_cfg.get('rank', 4))
        self.alpha = float(lora_cfg.get('alpha', 1.0))
        if not 1 <= self.rank <= 4:
            raise ValueError('LoRA rank must be in 1..4 (fused epilogue)')
        self.unet_lr = float(ucfg['lr'])
        H, W = self.latent_size
        probe_names = TrainEngine.lora_module_names.__get__(_NameProbe(self._topo, self.where))()
        if lora_state is None:
            lora_state = self._init_lora(probe_names)
        check_lora_ranks(lora_state, self.rank, 'unet')
        self.engine = TrainEngine(self._sd, self.batch, H, W, lora=lora_state, lora_alpha=self.alpha,
                                  attn_reg_weight=self.attn_reg_weight, reg_full_identity=self.reg_full_identity,
                                  lr=self.unet_lr, device=self.device, where=self.where, **self._topo)
        self._sd = None
        self.params_to_optimize_iterator = [{'params': [self.engine.state.params], 'lr': self.unet_lr}]

    def _init_lora(self, names):
        """LoRALinearLayer init (edlora.py:238-239): down ~ kaiming_uniform(a=sqrt(5)) (bound 1/sqrt(fan_in)), up = 0."""
        state = {}
        for m in names:
            w = self._sd[m + '.weight']
            N, K = w.shape[0], w.reshape(w.shape[0], -1).shape[1]
            bound = 1.0 / math.sqrt(K)
            state[f'{m}.lora_down.weight'] = (torch.rand(self.rank, K, generator=self._gen) * 2 - 1) * bound
            state[f'{m}.lora_up.weight'] = torch.zeros(N, self.rank)
        return state

    def get_params_to_optimize(self):
        return self.params_to_optimize_iterator

    def get_all_concept_token_ids(self):
        ids = []
        for _, cfg in self.new_concept_cfg.items():
            ids.extend(cfg['concept_token_ids'])
        return ids

    # ------------------------------------------------------------------------------------------ step
    def concept_token_positions(self, text_input_ids):
        """trainer_edlora.py:270-279 (host integers): positions of the concept tokens in each sample's layer-0 prompt."""
        b = self.batch
        ids = text_input_ids.reshape(b, -1, text_input_ids.shape[-1]).cpu()
        concept = set(int(i) for i in self.get_all_concept_token_ids())
        pos = []
        for text in ids:
            p = [i for i in range(text.shape[-1]) if int(text[0][i]) in concept]
            if len(p) != 2:
                raise ValueError(f'cal_attn_reg assumes exactly two concept tokens per prompt (:298), found {len(p)}')
            pos.append(p)
        return pos

    def forward(self, latents, encoder_hidden_states, masks, img_masks, text_input_ids=None, noise=None,
                timesteps=None, accumulate=False):
        """latents fp32 [b,4,h,w] (VAE output x 0.18215); encoder_hidden_states [b,16,77,768]; masks / img_masks
        [b,1,h,w].  noise / timesteps may be given (tests); otherwise sampled as trainer_edlora.py:207-214."""
        b = latents.shape[0]
        if b != self.batch:
            raise ValueError(f'batch {b} != batch_size_per_gpu {self.batch} the engine was built for')
        if noise is None:
            noise = torch.randn(latents.shape, generator=self._gen)
            if self.noise_offset is not None:
                noise = noise + self.noise_offset * torch.randn((b, latents.shape[1], 1, 1), generator=self._gen)
        if timesteps is None:
            timesteps = torch.randint(0, 1000, (b,), generator=self._gen)
        pos = None
        if self.attn_reg_weight is not None:
            if text_input_ids is None:
                raise ValueError('the attention regulariser needs text_input_ids to locate the concept tokens (:270)')
            pos = self.concept_token_positions(text_input_ids)
        loss_mask = masks if self.use_mask_loss else img_masks
        eng = self.engine
        n_layers = len(eng.xattn_names)
        out = eng.forward_backward(latents.to(self.device), noise.to(self.device), timesteps.to(self.device),
                                   ehs_to_layer_major(encoder_hidden_states.to(self.device), n_layers),
                                   masks.to(self.device), loss_mask=loss_mask.to(self.device), token_pos=pos,
                                   accumulate=accumulate)
        return out[0]

    __call__ = forward

    # ------------------------------------------------------------------------------------------ checkpoints
    def delta_state_dict(self):
        """trainer_edlora.py:358-378 layout; the text-side sections stay empty on this path."""
        delta = {'new_concept_embedding': {}, 'text_encoder': {}, 'unet': {}}
        for k, v in self.engine.lora_state_dict().items():
            v = v.cpu()
            delta['unet'][k] = v[:self.rank].clone() if k.endswith('lora_down.weight') else v[:, :self.rank].clone()
        return delta

    def load_delta_state_dict(self, delta_state_dict):
        """trainer_edlora.py:315-356 (unet section)."""
        unet = delta_state_dict.get('unet', {})
        if len(unet) == 0:
            return
        views = self.engine.lora_views
        if len(unet) != 2 * len(views):
            raise ValueError(f'checkpoint has {len(unet)} unet tensors, the model has {2 * len(views)} LoRA tensors')
        check_lora_ranks(unet, self.rank, 'unet')
        self.engine.load_lora_state_dict(unet)


class _NameProbe:
    """enough of the engine surface for TrainEngine.lora_module_names before the engine exists"""

    def __init__(self, topo, where='Attention'):
        from mos_b200.engine import cross_attention_names
        self.xattn_names = cross_attention_names(topo.get('block_out', (320, 640, 1280, 1280)), topo.get('layers', 2))
        self.where = where


# ================================================================================================ full ED-LoRA trainer
class EDLoRATrainer:
    """Reference constructor (trainer_edlora.py:21-68).  `pretrained_path`: diffusers-layout directory with unet/,
    text_encoder/ and tokenizer/.  Keyword extras of the GPU path (all optional, so that `EDLoRATrainer(**opt['models'])`
    works): `tokenizer` (an already constructed tokenizer), `latent_size`, `device`, `seed`.  `enable_xformers` /
    `gradient_checkpoint` are accepted and ignored (the attention kernels are this library's own; activations of one step
    fit HBM many times over)."""

    def __init__(self, pretrained_path, new_concept_token, initializer_token, enable_edlora, finetune_cfg=None,
                 noise_offset=None, attn_reg_weight=None, reg_full_identity=True, use_mask_loss=True,
                 enable_xformers=False, gradient_checkpoint=False, *, tokenizer=None, latent_size=(64, 64), device='cuda',
                 seed=0):
        from mixofshow.utils import model_io
        self.device = torch.device(device)
        self.enable_edlora = bool(enable_edlora)
        self.unet = model_io.load_unet(pretrained_path)                               # :44
        self.text_encoder = model_io.load_text_encoder(pretrained_path, device=device)   # :41
        if tokenizer is None:
            from transformers import CLIPTokenizer
            tokenizer = CLIPTokenizer.from_pretrained(pretrained_path, subfolder='tokenizer')   # :40
        self.tokenizer = tokenizer
        import os
        self.vae = model_io.load_vae(pretrained_path, device=device) if os.path.isdir(os.path.join(pretrained_path, 'vae')) \
            else None                                                                     # :39
        self._gen = torch.Generator(device='cpu').manual_seed(seed)
        self.new_concept_cfg = self.init_new_concept(new_concept_token, initializer_token,
                                                     enable_edlora=self.enable_edlora)   # :55
        self.attn_reg_weight = attn_reg_weight
        self.reg_full_identity = reg_full_identity
        self.noise_offset = noise_offset
        self.use_mask_loss = use_mask_loss
        self.latent_size = tuple(latent_size)
        self.engine = self.text_engine = self.state = None
        self._batch = None
        self._loaded = None
        if finetune_cfg:
            self.set_finetune_cfg(finetune_cfg)

    # ------------------------------------------------------------------------------------------ new concept tokens
    def init_new_concept(self, new_concept_tokens, initializer_tokens, enable_edlora=True):
        """trainer_edlora.py:144-194: 16 tokens `<new{k}>` per concept word (1 without ED-LoRA), embedding rows initialised from
        `<rand-sigma>` or from an existing single token."""
        new_concept_cfg = {}
        new_concept_tokens = new_concept_tokens.split('+')
        if initializer_tokens is None:
            initializer_tokens = ['<rand-0.017>'] * len(new_concept_tokens)
        else:
            initializer_tokens = initializer_tokens.split('+')
        assert len(new_concept_tokens) == len(initializer_tokens), 'concept token should match init token.'
        for idx, (concept_name, init_token) in enumerate(zip(new_concept_tokens, initializer_tokens)):
            num_new_embedding = 16 if enable_edlora else 1
            new_token_names = [f'<new{idx * num_new_embedding + layer_id}>' for layer_id in range(num_new_embedding)]
            num_added_tokens = self.tokenizer.add_tokens(new_token_names)
            assert num_added_tokens == len(new_token_names), 'some token is already in tokenizer'
            new_token_ids = [self.tokenizer.convert_tokens_to_ids(token_name) for token_name in new_token_names]
            self.text_encoder.resize_token_embeddings(len(self.tokenizer))
            token_embeds = self.text_encoder.get_input_embeddings().weight.data
            if init_token.startswith('<rand'):
                sigma_val = float(re.findall(r'<rand-(.*)>', init_token)[0])
                init_feature = torch.randn(token_embeds[0].shape, generator=self._gen) * sigma_val
            else:
                init_token_ids = self.tokenizer.encode(init_token, add_special_tokens=False)
                if len(init_token_ids) > 1 or init_token_ids[0] == 40497:        # sic, :179
                    raise ValueError('The initializer token must be a single existing token.')
                init_feature = token_embeds[init_token_ids[0]]
            for token_id in new_token_ids:
                token_embeds[token_id] = init_feature.clone()
            new_concept_cfg.update({concept_name: {'concept_token_ids': new_token_ids,
                                                   'concept_token_names': new_token_names}})
        return new_concept_cfg

    def get_all_concept_token_ids(self):
        ids = []
        for _, cfg in self.new_concept_cfg.items():
            ids.extend(cfg['concept_token_ids'])
        return ids

    # ------------------------------------------------------------------------------------------ configuration
    def set_finetune_cfg(self, finetune_cfg):
        """trainer_edlora.py:70-142: up to three parameter groups with their own learning rates.  A group trains iff its
        `enable_tuning` is set (and, for the LoRA groups, a `lora_cfg` is given, :97 / :118); at least one must."""
        te, tx, un = (finetune_cfg.get(k) or {} for k in FINETUNE_GROUPS)
        self.train_emb = bool(te.get('enable_tuning'))
        self.train_text = bool(tx.get('enable_tuning') and tx.get('lora_cfg'))
        self.train_unet = bool(un.get('enable_tuning') and un.get('lora_cfg'))
        if not (self.train_emb or self.train_text or self.train_unet):
            raise ValueError('finetune_cfg enables no parameter group: set enable_tuning on text_embedding, text_encoder '
                             '(with a lora_cfg) or unet (with a lora_cfg)')
        self.text_where = self.unet_where = None
        self.text_rank = self.unet_rank = 4
        self.text_alpha = self.unet_alpha = 1.0
        if self.train_emb and 'weight_decay' in te:
            raise NotImplementedError('a per-group weight_decay for the embeddings is not supported by the flat AdamW')
        if self.train_text:
            tcfg = dict(tx['lora_cfg'])
            self.text_where = _check_where(tcfg.pop('where'), CLIP_WHERE, 'text_encoder')
            self.text_rank, self.text_alpha = _check_rank(tcfg)
        if self.train_unet:
            ucfg = dict(un['lora_cfg'])
            self.unet_where = _check_where(ucfg.pop('where'), UNET_WHERE, 'unet')
            self.unet_rank, self.unet_alpha = _check_rank(ucfg)
        self.groups = tuple(g for g, on in zip(FINETUNE_GROUPS, (self.train_emb, self.train_text, self.train_unet)) if on)
        # the flat state keeps three learning-rate slots; an absent group has zero length and its slot is never read
        self.lrs = tuple(float(c['lr']) if on else 0.0
                         for c, on in zip((te, tx, un), (self.train_emb, self.train_text, self.train_unet)))
        self.params_to_optimize_iterator = [{'lr': lr} for g, lr in zip(FINETUNE_GROUPS, self.lrs) if g in self.groups]

    def get_params_to_optimize(self):
        return self.params_to_optimize_iterator

    # ------------------------------------------------------------------------------------------ engines
    def _kaiming(self, rank, K):
        return (torch.rand(rank, K, generator=self._gen) * 2 - 1) / math.sqrt(K)       # edlora.py:238

    def _topology(self):
        c = self.unet.config
        return dict(block_out=tuple(c.block_out_channels), layers=c.layers_per_block, heads=c.attention_head_dim,
                    cross_dim=c.cross_attention_dim)

    def lora_module_names(self):
        """{'text_encoder': [...], 'unet': [...]}: the modules that carry a LoRA (trainer_edlora.py:100-133), empty for a
        group that does not train"""
        from mos_b200.clip_train_engine import CLIPTrainEngine
        names = {'text_encoder': [], 'unet': []}
        if self.train_text:
            names['text_encoder'] = CLIPTrainEngine.module_names(_n_layers(self.text_encoder.state_dict()), self.text_where)
        if self.train_unet:
            probe = _NameProbe(self._topology(), self.unet_where)
            names['unet'] = TrainEngine.lora_module_names.__get__(probe)()
        return names

    def flat_group_sizes(self):
        """floats of the three groups of the flat training state [concept rows | text LoRA | UNet LoRA] (0 = absent);
        the LoRA blocks keep rank-4 slots and the text encoder's GEMM pads"""
        from mos_b200.clip_train_engine import CLIPTrainEngine
        tsd = self.text_encoder.state_dict()
        C = tsd['text_model.embeddings.token_embedding.weight'].shape[1]
        n_text = 0
        if self.train_text:
            heads = getattr(self.text_encoder, 'hf_config', {}).get('num_attention_heads', 12)
            n_inner = tsd['text_model.encoder.layers.0.mlp.fc1.weight'].shape[0]
            n_text = CLIPTrainEngine.lora_param_count(_n_layers(tsd), C, heads * 80, where=self.text_where, inner=n_inner)
        names = self.lora_module_names()
        usd = self.unet.state_dict()
        n_unet = sum(4 * (usd[m + '.weight'].reshape(usd[m + '.weight'].shape[0], -1).shape[1] + usd[m + '.weight'].shape[0])
                     for m in names['unet'])
        n_rows = len(self.get_all_concept_token_ids()) if self.train_emb else 0
        return n_rows * C, n_text, n_unet

    def _build(self, batch):
        from mos_b200.clip_engine import CLIPTextEngine
        from mos_b200.clip_train_engine import CLIPTrainEngine
        from mos_b200.dp import FlatTrainState
        topo = self._topology()
        usd = {k: v.detach() for k, v in self.unet.state_dict().items()}
        tsd = self.text_encoder.state_dict()
        names = self.lora_module_names()
        unet_names, text_names = names['unet'], names['text_encoder']
        ulora, tlora = {}, {}
        for m in unet_names:                                   # LoRALinearLayer init: down kaiming, up zeros (:238-239)
            w = usd[m + '.weight']
            ulora[f'{m}.lora_down.weight'] = self._kaiming(self.unet_rank, w.reshape(w.shape[0], -1).shape[1])
            ulora[f'{m}.lora_up.weight'] = torch.zeros(w.shape[0], self.unet_rank)
        for m in text_names:
            w = tsd[m + '.weight']
            tlora[f'{m}.lora_down.weight'] = self._kaiming(self.text_rank, w.shape[1])
            tlora[f'{m}.lora_up.weight'] = torch.zeros(w.shape[0], self.text_rank)
        ids = self.get_all_concept_token_ids()
        C = tsd['text_model.embeddings.token_embedding.weight'].shape[1]
        heads = getattr(self.text_encoder, 'hf_config', {}).get('num_attention_heads', 12)
        _, n_text, n_unet = self.flat_group_sizes()
        self.state = FlatTrainState(len(ids) if self.train_emb else 0, C, n_text, n_unet, lrs=self.lrs, device=self.device)
        text_grad = self.train_emb or self.train_text
        H, W = self.latent_size
        self.engine = TrainEngine(usd, batch, H, W, lora=ulora if self.train_unet else None, lora_alpha=self.unet_alpha,
                                  attn_reg_weight=self.attn_reg_weight, reg_full_identity=self.reg_full_identity,
                                  state=self.state, state_offset=self.state.group_end[1], text_grad=text_grad,
                                  device=self.device, where=self.unet_where or UNET_WHERE[0],
                                  shared_ehs=not self.enable_edlora, **topo)
        n_x = len(self.engine.xattn_names) if self.enable_edlora else 1      # text sequences per sample
        if text_grad:
            self.text_engine = CLIPTrainEngine(tsd, n_x * batch, lora=tlora if self.train_text else None,
                                               lora_alpha=self.text_alpha, concept_token_ids=ids, state=self.state,
                                               emb_offset=0 if self.train_emb else None,
                                               lora_offset=self.state.group_end[0], device=self.device, heads=heads,
                                               where=self.text_where or CLIP_WHERE[0])
        else:                       # UNet only: the text encoder (concept rows included) is a constant forward
            self.text_engine = CLIPTextEngine(tsd, n_x * batch, device=self.device, heads=heads)
        self._rows_dev = torch.tensor(ids, dtype=torch.long, device=self.device)
        if not self.train_emb and ids:
            self.state.set_const_rows(self._concept_rows())
        self.engine.attach_text_engine(self.text_engine)
        self._batch = batch
        if self._loaded is not None:
            self._apply_delta(self._loaded)
            self._loaded = None

    def _concept_rows(self):
        """the current new-concept rows fp32 [R, 768] on the device (trained, or constants of the token table)"""
        if self.train_emb:
            return self.text_engine.emb_view
        return self.text_engine.tok[self._rows_dev]

    # ------------------------------------------------------------------------------------------ step
    def tokenize_layerwise(self, prompts):
        """prompts (b strings) -> token ids [(b 16), 77] as the reference builds them (:223-231) and the same ids in the
        engines' layer-major order [16 * b, 77]."""
        from mixofshow.pipelines.pipeline_edlora import bind_concept_prompt
        bound = bind_concept_prompt(list(prompts), new_concept_cfg=self.new_concept_cfg)
        ids = self.tokenizer(bound, padding='max_length', max_length=self.tokenizer.model_max_length, truncation=True,
                             return_tensors='pt').input_ids
        b = len(prompts)
        n_x = ids.shape[0] // b
        return ids, ids.view(b, n_x, -1).permute(1, 0, 2).reshape(n_x * b, -1).contiguous()

    def tokenize(self, prompts):
        """vanilla LoRA (:220-231 without the binding): prompts (b strings) -> token ids [b, 77], as written"""
        return self.tokenizer(list(prompts), padding='max_length', max_length=self.tokenizer.model_max_length,
                              truncation=True, return_tensors='pt').input_ids

    def concept_token_positions(self, ids, b):
        """trainer_edlora.py:270-279: the positions of the concept tokens in each sample's first id row (ids [(b l), 77],
        l = 16 layer prompts with ED-LoRA, 1 without); the regulariser needs exactly two per sample"""
        concept = set(int(i) for i in self.get_all_concept_token_ids())
        pos = []
        for text in ids.view(b, -1, ids.shape[-1]):
            p = [i for i in range(text.shape[-1]) if int(text[0][i]) in concept]
            if len(p) != 2:
                raise ValueError(f'cal_attn_reg assumes exactly two concept tokens per prompt (:298), found {len(p)}')
            pos.append(p)
        return pos

    def forward(self, images, prompts, masks, img_masks, noise=None, timesteps=None, accumulate=False):
        """trainer_edlora.py:202-261.  `images`: [b,3,H,W] in [-1,1] (encoded by the GPU VAE, :203-204) or already encoded
        latents [b,4,h,w] (x 0.18215).  Runs forward + loss + backward of the whole step (text encoder and UNet) and returns
        the loss as a device scalar."""
        if images.shape[1] == 3:                  # :203-204: latents = vae.encode(images).latent_dist.sample() * 0.18215
            if self.vae is None:
                raise ValueError(f'images were given but the model directory has no vae/: pass latents [b,4,h,w] (x 0.18215)')
            dist = self.vae.encode(images.to(self.device)).latent_dist
            latents = (dist.mean + dist.std * torch.randn(dist.mean.shape, generator=self._gen).to(self.device)) * 0.18215
        else:
            latents = images
        b = latents.shape[0]
        if self.engine is None:
            self._build(b)
        if b != self._batch:
            raise ValueError(f'batch {b} != the batch {self._batch} the engines were built for')
        if noise is None:
            noise = torch.randn(latents.shape, generator=self._gen)
            if self.noise_offset is not None:
                noise = noise + self.noise_offset * torch.randn((b, latents.shape[1], 1, 1), generator=self._gen)
        if timesteps is None:
            timesteps = torch.randint(0, 1000, (b,), generator=self._gen)
        if self.enable_edlora:
            ids, ids_lm = self.tokenize_layerwise(prompts)
        else:
            ids = ids_lm = self.tokenize(prompts)
        n_x = len(self.engine.xattn_names)
        if self.enable_edlora and ids.shape[0] // b != n_x:          # a smaller topology uses the first n_x layer prompts of every sample
            ids_lm = ids.view(b, -1, ids.shape[-1])[:, :n_x].permute(1, 0, 2).reshape(n_x * b, -1).contiguous()
        pos = self.concept_token_positions(ids, b) if self.attn_reg_weight is not None else None
        loss_mask = masks if self.use_mask_loss else img_masks
        dev = self.device
        out = self.engine.forward_backward(latents.to(dev), noise.to(dev), timesteps.to(dev), None, masks.to(dev),
                                           loss_mask=loss_mask.to(dev), token_pos=pos, accumulate=accumulate,
                                           text_ids=ids_lm)
        return out[0]

    __call__ = forward

    def refresh(self):
        """after an optimiser step on the flat state: re-pack the LoRA sets and write the embedding rows back (a frozen
        group issues nothing)"""
        self.engine.refresh_lora()
        if self.train_emb or self.train_text:
            self.text_engine.refresh_lora()

    # ------------------------------------------------------------------------------------------ checkpoints
    def delta_state_dict(self):
        """trainer_edlora.py:358-378: the concept rows always (trained or not), the LoRAs of the groups that train (an
        absent group leaves its section empty)."""
        if self.engine is None:
            raise RuntimeError('delta_state_dict before the first forward: the engines are built on the first batch')
        delta = {'new_concept_embedding': {}, 'text_encoder': {}, 'unet': {}}
        rows = self._concept_rows().detach().cpu()
        k = 0
        for concept_name, cfg in self.new_concept_cfg.items():
            n = len(cfg['concept_token_ids'])
            delta['new_concept_embedding'][concept_name] = rows[k:k + n].clone()
            k += n
        for key, v in (self.text_engine.lora_state_dict() if self.train_text else {}).items():
            v = v.cpu()
            delta['text_encoder'][key] = (v[:self.text_rank] if key.endswith('lora_down.weight') else v[:, :self.text_rank]).clone()
        for key, v in self.engine.lora_state_dict().items():
            v = v.cpu()
            delta['unet'][key] = (v[:self.unet_rank] if key.endswith('lora_down.weight') else v[:, :self.unet_rank]).clone()
        return delta

    def load_delta_state_dict(self, delta_state_dict):
        """trainer_edlora.py:315-356 (applied when the engines exist, i.e. at the first batch at the latest).  Unlike the
        reference, which skips the LoRA tensors of a group it does not train (no parameter name matches them), a checkpoint
        carrying a LoRA for such a group is refused with ValueError rather than silently half-loaded, and so is a LoRA
        whose rank is not the configured rank of its group (check_lora_ranks), before any engine is touched."""
        for part, on, rank in (('text_encoder', self.train_text, self.text_rank), ('unet', self.train_unet, self.unet_rank)):
            if on:
                check_lora_ranks(delta_state_dict.get(part) or {}, rank, part)
        if self.engine is None:
            self._loaded = delta_state_dict
        else:
            self._apply_delta(delta_state_dict)

    def _apply_delta(self, delta):
        emb = delta.get('new_concept_embedding') or {}
        if emb:
            rows = self._concept_rows().clone()
            k = 0
            for concept_name, cfg in self.new_concept_cfg.items():
                n = len(cfg['concept_token_ids'])
                if concept_name in emb:
                    rows[k:k + n] = emb[concept_name].to(self.device, torch.float32)
                k += n
            if self.train_emb:
                self.text_engine.emb_view.copy_(rows)
            else:                   # constants of the text encoder (and of the Norm_mean state)
                self.text_engine.tok.index_copy_(0, self._rows_dev, rows)
                if self.state.const_rows is not None:
                    self.state.set_const_rows(rows)
        for part, on, eng in (('text_encoder', self.train_text, self.text_engine), ('unet', self.train_unet, self.engine)):
            if not delta.get(part):
                continue
            if not on:
                raise ValueError(f'the checkpoint has a {part} LoRA but finetune_cfg does not train that group')
            eng.load_lora_state_dict(delta[part])
        self.refresh()
