"""Loader of the input-resolution fixtures (oracle/make_resize_golden.py): one TimeSformer per attention type,
fed clips whose patch grid differs from the one img_size built, with the reference's outputs and gradients per case."""
from __future__ import annotations

import torch

from tests.conftest import load_golden

FAMILIES = {'resize_divided': 'divided_space_time', 'resize_space_only': 'space_only',
            'resize_joint': 'joint_space_time'}
CASES = {'resize_divided': ['up48', 'down16', 'h48w64', 'h64w48', 'fixed_h48w64', 'big272'],
         'resize_space_only': ['up48', 'down16', 'h48w64', 'h64w48', 'fixed_h48w64'],
         'resize_joint': ['up48', 'down16', 'h48w64', 'h64w48', 'fixed_h48w64']}
PARAMS = [(f, t) for f, tags in CASES.items() for t in tags]


class ResizeCase:
    """One input size of a family: x, the reference's eval / train outputs and gradients (.grad / .gradsum as
    tests.conftest.check_grads reads them)."""

    def __init__(self, z, tag):
        self.tag = tag
        h, w, B, learnable, seed = (int(v) for v in z[f'meta::{tag}'])
        self.size, self.B, self.learnable, self.train_seed = (h, w), B, bool(learnable), seed
        self.x = torch.from_numpy(z[f'xq::{tag}']).float() / 32          # exact in fp32
        self.y_eval = torch.from_numpy(z[f'out::{tag}::y_eval'])
        self.y_train = torch.from_numpy(z[f'out::{tag}::y_train'])
        self.loss_w = torch.linspace(-1, 1, self.y_train.numel(), dtype=torch.float64).reshape(self.y_train.shape)
        self.grad = {k.split('::', 2)[2]: torch.from_numpy(z[k]) for k in z if k.startswith(f'grad::{tag}::')}
        self.gradsum = {k.split('::', 2)[2]: z[k] for k in z if k.startswith(f'gradsum::{tag}::')}


class ResizeFamily:
    def __init__(self, name):
        z = load_golden(name)
        self.name = name
        self.attention_type = FAMILIES[name]
        self.cfg = {k[4:]: int(z[k]) for k in z if k.startswith('cfg_')}
        self.sd = {k[4:]: torch.from_numpy(z[k]) for k in z if k.startswith('sd::')}
        self.cases = {str(t): ResizeCase(z, str(t)) for t in z['cases']}

    def model(self, learnable=True):
        from videotransformer_pytorch_b200 import TimeSformer
        c = self.cfg
        m = TimeSformer(num_frames=c['num_frames'], img_size=c['img_size'], patch_size=c['patch_size'],
                        embed_dims=c['embed_dims'], num_heads=c['num_heads'],
                        num_transformer_layers=c['num_transformer_layers'], attention_type=self.attention_type,
                        use_learnable_pos_emb=learnable)
        sd = self.sd if learnable else {k: v for k, v in self.sd.items() if k not in ('pos_embed', 'time_embed')}
        m.load_state_dict(sd, strict=True)
        return m


_CACHE = {}


def family(name):
    if name not in _CACHE:
        _CACHE[name] = ResizeFamily(name)
    return _CACHE[name]
