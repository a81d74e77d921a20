"""Attention controllers with the reference's call protocol (mixofshow/utils/ptp_util.py:11-108): the GPU processors
hand them the cross-attention probability maps `[B*heads, N, 77]`.  Notebook visualisation helpers of the reference
file are out of scope (SURVEY.md §2.1 row 8)."""
import abc


class EmptyControl:
    def step_callback(self, x_t):
        return x_t

    def between_steps(self):
        return

    def __call__(self, attn, is_cross: bool, place_in_unet: str):
        return attn


class AttentionControl(abc.ABC):
    """Counts attention layers; after `num_att_layers` calls a denoise step is complete (ptp_util.py:37-53)."""

    def __init__(self, low_resource, training):
        self.cur_step = 0
        self.num_att_layers = -1
        self.cur_att_layer = 0
        self.low_resource = low_resource
        self.training = training

    def step_callback(self, x_t):
        return x_t

    def between_steps(self):
        return

    @property
    def num_uncond_att_layers(self):
        return self.num_att_layers if self.low_resource else 0

    @abc.abstractmethod
    def forward(self, attn, is_cross: bool, place_in_unet: str):
        raise NotImplementedError

    def __call__(self, attn, is_cross: bool, place_in_unet: str):
        if self.cur_att_layer >= self.num_uncond_att_layers:
            if self.low_resource or self.training:
                attn = self.forward(attn, is_cross, place_in_unet)      # training: the whole [B*8, N, 77] tensor
            else:
                h = attn.shape[0]                                        # sampling: conditional half only
                attn[h // 2:] = self.forward(attn[h // 2:], is_cross, place_in_unet)
        self.cur_att_layer += 1
        if self.cur_att_layer == self.num_att_layers + self.num_uncond_att_layers:
            self.cur_att_layer = 0
            self.cur_step += 1
            self.between_steps()
        return attn

    def reset(self):
        self.cur_step = 0
        self.cur_att_layer = 0


class AttentionStore(AttentionControl):
    """Accumulates the maps per place ('down' | 'mid' | 'up') x ('cross' | 'self') over steps (ptp_util.py:67-108)."""
    PLACES = ('down_cross', 'mid_cross', 'up_cross', 'down_self', 'mid_self', 'up_self')

    def __init__(self, low_resource=False, training=False):
        super().__init__(low_resource, training)
        self.step_store = self.get_empty_store()
        self.attention_store = {}

    @staticmethod
    def get_empty_store():
        return {k: [] for k in AttentionStore.PLACES}

    def forward(self, attn, is_cross: bool, place_in_unet: str):
        self.step_store[f"{place_in_unet}_{'cross' if is_cross else 'self'}"].append(attn)
        return attn

    def between_steps(self):
        if len(self.attention_store) == 0:
            self.attention_store = self.step_store
        else:
            for key, maps in self.attention_store.items():
                for i in range(len(maps)):
                    maps[i] = maps[i] + self.step_store[key][i]
        self.step_store = self.get_empty_store()

    def get_average_attention(self):
        return {key: [m / self.cur_step for m in maps] for key, maps in self.attention_store.items()}

    def reset(self):
        super().reset()
        self.step_store = self.get_empty_store()
        self.attention_store = {}
