"""SeisT (Seismogram Transformer) behind the reference's `@register_model` surface, executed by
hand-written sm_90a CUDA kernels.

What is kept from the reference (models/seist.py): the registered creator names
(:940-1170), the hyper-parameter presets (:855-937), and the *parameter tree* — every
nn.Conv1d / nn.BatchNorm1d / nn.Linear lives at the same attribute path, so `state_dict()` keys,
shapes and dtypes are identical (SURVEY §3.4) and the reference's `pretrained/*.pth` load with
`strict=True`.  What is not kept: the modules below are parameter holders only.  `forward` does
not dispatch ~480 leaf modules (:833-852); it runs a pre-compiled plan of fused CUDA kernels
(seist_b200/plan.py, seist_b200/csrc) over one flat parameter buffer.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List

import torch
import torch.nn as nn

from ._factory import register_model

__all__: List[str] = []


# ------------------------------------------------------------------------------------------------
# hyper-parameters
# ------------------------------------------------------------------------------------------------
@dataclass
class HParams:
    """Constructor arguments of the reference `SeismogramTransformer` (models/seist.py:618-645)."""
    in_channels: int = 3
    stem_channels: List[int] = field(default_factory=lambda: [16, 8, 16, 16])
    stem_kernel_sizes: List[int] = field(default_factory=lambda: [11, 5, 5, 7])
    stem_strides: List[int] = field(default_factory=lambda: [2, 1, 1, 2])
    layer_blocks: List[int] = field(default_factory=lambda: [2, 3, 6, 2])
    layer_channels: List[int] = field(default_factory=lambda: [24, 32, 64, 96])
    attn_blocks: List[int] = field(default_factory=lambda: [1, 1, 2, 1])
    stage_aggr_ratios: List[int] = field(default_factory=lambda: [2, 2, 2, 2])
    attn_aggr_ratios: List[int] = field(default_factory=lambda: [8, 4, 2, 1])
    head_dims: List[int] = field(default_factory=lambda: [8, 8, 16, 32])
    msmc_kernel_sizes: List[int] = field(default_factory=lambda: [3, 5])
    path_drop_rate: float = 0.2
    attn_drop_rate: float = 0.1
    key_drop_rate: float = 0.1
    mlp_drop_rate: float = 0.2
    other_drop_rate: float = 0.1
    attn_ratio: float = 0.6
    mlp_ratio: int = 2
    qkv_bias: bool = True
    mlp_bias: bool = True
    # output head: "dpk" (HeadDetectionPicking :507), "reg" (HeadRegression :594), "cls" (:575)
    head: str = "dpk"
    head_out_channels: int = 3
    head_scale: float = 1.0
    head_num_classes: int = 2
    head_sigmoid: bool = True   # dpk out_act: Sigmoid (registered variants) vs Identity (class default)


def round_channels(v: int, divisor: int) -> int:
    """Nearest multiple of `divisor` not more than 10 % below v (reference `_make_divisible`, :51-60)."""
    r = max(divisor, (int(v + divisor / 2) // divisor) * divisor)
    return r + divisor if r < 0.9 * v else r


def same_pad(length: int, k: int, stride: int):
    """(left, right) zeros so a stride-`stride` conv emits ceil(length/stride) samples; the odd
    sample goes right (reference `_auto_pad_1d`, :12-48)."""
    if k < stride:
        raise AssertionError(f"`kernel_size` must be greater than or equal to `stride`, got {k}, {stride}")
    total = (stride - length % stride) % stride + k - stride
    return total // 2, total - total // 2


def split_msmc(io_dim: int, groups: int, n_paths: int) -> List[int]:
    """Channel split of MultiScaleMixedConv (:274-285)."""
    gsize = io_dim // groups
    dims: List[int] = []
    while len(dims) < n_paths:
        d = round_channels((io_dim - sum(dims)) // (n_paths - len(dims)), gsize)
        assert d > 0
        dims.append(d)
    return dims


def split_mptl(io_dim: int, attn_ratio: float, head_dim: int):
    """(attention channels, conv channels) of MultiPathTransformerLayer (:420-423)."""
    a = round_channels(int(io_dim * attn_ratio), head_dim) if attn_ratio > 0 else 0
    return a, max(io_dim - a, 0)


def dpk_head_layers(hp: HParams):
    """[(cin, cout, k)] of the up-sampling head, derived from every stride>1 stage (:777-793,:529-536)."""
    feats = [hp.in_channels] + hp.stem_channels + hp.layer_channels[:-1]
    kers = hp.stem_kernel_sizes + [max(hp.msmc_kernel_sizes)] * len(hp.layer_channels)
    strides = hp.stem_strides + hp.stage_aggr_ratios
    picked = [(c, k) for c, k, s in zip(feats, kers, strides) if s > 1][::-1]
    chans = [c for c, _ in picked]
    ins = [hp.layer_channels[-1]] + chans[:-1]
    outs = chans[:-1] + [hp.head_out_channels * 2]
    return [(i, o, k) for i, o, (_, k) in zip(ins, outs, picked)]


def dpk_up_sizes(l_in: int, l_out: int, depth: int) -> List[int]:
    """Per-layer interpolation targets (:554-559): geometric steps, truncated from the top down."""
    sizes = [l_out] * depth
    f = (l_out / l_in) ** (1 / depth)
    for i in reversed(range(depth - 1)):
        sizes[i] = int(sizes[i + 1] / f)
    return sizes


# ------------------------------------------------------------------------------------------------
# parameter tree (holders only — no forward of their own)
# ------------------------------------------------------------------------------------------------
class _Node(nn.Module):
    """Pure container; children are attached by the builders below."""


def _conv(cin, cout, k=1, stride=1, groups=1, bias=False, padding=0):
    return nn.Conv1d(cin, cout, k, stride=stride, groups=groups, bias=bias, padding=padding)


def _mlp(dim, ratio, bias):
    n = _Node()
    n.lin0 = _conv(dim, int(dim * ratio), bias=bias)
    n.lin1 = _conv(int(dim * ratio), dim, bias=bias)
    return n


def _aggr(cin, cout):
    n = _Node()
    n.proj = _conv(cin, cout)
    n.norm = nn.BatchNorm1d(cout)
    return n


def _stem_path(cin, cout, k, stride):
    n = _Node()
    n.in_proj = _conv(cin, cin)
    n.dconv = _conv(cin, cin, k, stride=stride, groups=cin)
    n.pconv = _conv(cin, cout)
    n.norm = nn.BatchNorm1d(cout)
    return n


def _stem_block(cin, cout, k, stride, npath=3):
    n = _Node()
    n.convs = nn.ModuleList([_stem_path(cin, cout, k + 4 * p, stride) for p in range(npath)])
    n.out_proj = _conv(npath * cout, cout)
    n.norm = nn.BatchNorm1d(cout)
    return n


def _gconv_block(dim, groups, k, hp: HParams):
    n = _Node()
    n.conv = _conv(dim, dim, k, groups=groups)
    n.norm0 = nn.BatchNorm1d(dim)
    n.proj = _conv(dim, dim)
    n.norm1 = nn.BatchNorm1d(dim)
    n.mlp = _mlp(dim, hp.mlp_ratio, hp.mlp_bias)
    return n


def _msmc(io_dim, groups, hp: HParams):
    n = _Node()
    gsize = io_dim // groups
    dims = split_msmc(io_dim, groups, len(hp.msmc_kernel_sizes))
    n.projs = nn.ModuleList([_conv(io_dim, d) for d in dims])
    n.norms = nn.ModuleList([nn.BatchNorm1d(d) for d in dims])
    n.convs = nn.ModuleList([_gconv_block(d, d // gsize, k, hp) for d, k in zip(dims, hp.msmc_kernel_sizes)])
    n.out_norm = nn.BatchNorm1d(io_dim)
    return n


def _attention(dim, aggr_ratio, hp: HParams):
    n = _Node()
    if aggr_ratio > 1:
        n.aggr = _aggr(dim, dim)
        n.norm = nn.BatchNorm1d(dim)
    for name in ("q_proj", "k_proj", "v_proj", "out_proj"):
        setattr(n, name, _conv(dim, dim, bias=hp.qkv_bias))
    return n


def _mptl(io_dim, head_dim, aggr_ratio, hp: HParams):
    n = _Node()
    a_dim, c_dim = split_mptl(io_dim, hp.attn_ratio, head_dim)
    if a_dim > 0:
        n.attn_proj = _conv(io_dim, a_dim)
        n.norm0 = nn.BatchNorm1d(a_dim)
        n.attention = _attention(a_dim, aggr_ratio, hp)
    if c_dim > 0:
        n.conv_proj = _conv(io_dim, c_dim)
        n.norm1 = nn.BatchNorm1d(c_dim)
        n.gconv = _gconv_block(c_dim, c_dim // head_dim, 3, hp)
    n.norm2 = nn.BatchNorm1d(io_dim)
    n.mlp = _mlp(io_dim, hp.mlp_ratio, hp.mlp_bias)
    return n


def _dpk_head(hp: HParams):
    n = _Node()
    ups = []
    for cin, cout, k in dpk_head_layers(hp):
        u = nn.Sequential()
        u.add_module("conv", _conv(cin, cout, k, bias=True))
        u.add_module("norm", nn.BatchNorm1d(cout))
        ups.append(u)
    n.up_layers = nn.ModuleList(ups)
    n.out_conv = _conv(hp.head_out_channels * 2, hp.head_out_channels, 7, bias=True, padding=3)
    return n


def _vec_head(hp: HParams):
    n = _Node()
    n.lin = nn.Linear(hp.layer_channels[-1], 1 if hp.head == "reg" else hp.head_num_classes)
    return n


class SeismogramTransformer(nn.Module):
    """Drop-in for the reference class of the same name (models/seist.py:613-852).

    `forward(x)`: x float32 (N, in_channels, L) on a CUDA device -> (N, 3, L) probabilities (dpk)
    or (N, 1) / (N, classes) (reg / cls).  train()/eval() switch BatchNorm between batch and
    running statistics and dropout on/off exactly as torch modules do.  There is no CPU path.
    """

    def __init__(self, hp: HParams | None = None, **kwargs):
        super().__init__()
        kwargs.pop("in_samples", None)        # swallowed by **kwargs in the reference too (:644)
        hp = hp or HParams()
        for key, val in kwargs.items():
            if not hasattr(hp, key):
                raise TypeError(f"unexpected argument {key!r}")
            setattr(hp, key, val)
        lens = {len(hp.layer_blocks), len(hp.layer_channels), len(hp.stage_aggr_ratios),
                len(hp.attn_aggr_ratios), len(hp.attn_blocks), len(hp.head_dims)}
        assert len(lens) == 1 and len(hp.stem_channels) == len(hp.stem_kernel_sizes) == len(hp.stem_strides)
        self.hp = hp

        cins = [hp.in_channels] + hp.stem_channels[:-1]
        self.stem = nn.Sequential(*[
            _stem_block(ci, co, k, s)
            for ci, co, k, s in zip(cins, hp.stem_channels, hp.stem_kernel_sizes, hp.stem_strides)])

        self.encoder_layers = nn.ModuleList()
        prev = hp.stem_channels[-1]
        for i, lc in enumerate(hp.layer_channels):
            mods = [_aggr(prev, lc)]
            n_conv = hp.layer_blocks[i] - hp.attn_blocks[i]
            for j in range(hp.layer_blocks[i]):
                if j >= n_conv:
                    mods.append(_mptl(lc, hp.head_dims[i], hp.attn_aggr_ratios[i], hp))
                else:
                    mods.append(_msmc(lc, lc // hp.head_dims[i], hp))
            self.encoder_layers.append(nn.Sequential(*mods))
            prev = lc

        self.out_head = _dpk_head(hp) if hp.head == "dpk" else _vec_head(hp)
        self.reset_parameters()
        self._engine = None

    # -- initialisation (reference `_init_weights`, :816-831) -------------------------------------
    def reset_parameters(self):
        for m in self.modules():
            if isinstance(m, (nn.Conv1d, nn.Linear)):
                nn.init.trunc_normal_(m.weight, std=0.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
            elif isinstance(m, nn.modules.batchnorm._BatchNorm):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)

    def block_drop_path_rates(self) -> List[float]:
        """Linear stochastic-depth schedule over all blocks (:705)."""
        return [v.item() for v in torch.linspace(0, self.hp.path_drop_rate, sum(self.hp.layer_blocks))]

    def set_drop_rates(self, **rates):
        """Change path/attn/key/mlp/other drop rates after construction (plans are rebuilt)."""
        for k, v in rates.items():
            assert k in ("path_drop_rate", "attn_drop_rate", "key_drop_rate", "mlp_drop_rate", "other_drop_rate")
            setattr(self.hp, k, float(v))
        if self._engine is not None:
            self._engine.invalidate()
        return self

    # -- execution ---------------------------------------------------------------------------------
    def engine(self):
        if self._engine is None:
            from ..engine import Engine
            self._engine = Engine(self)
        return self._engine

    @torch._dynamo.disable
    def forward(self, x):
        # `torch.compile(model)` (the reference's default, training/train.py:296-297) degrades to a graph break here:
        # the forward is one opaque call into the C-ABI plan executor, there is nothing for Inductor to fuse
        if not x.is_cuda:
            raise RuntimeError("seist_b200 has no CPU path: the input must live on a CUDA (sm_90a) device")
        return self.engine().forward(x)

    def _apply(self, fn, *args, **kwargs):
        # .to()/.cuda()/.float() re-create parameter storage: drop the flat buffers and plans.
        if getattr(self, "_engine", None) is not None:
            self._engine.invalidate(release_flat=True)
        return super()._apply(fn, *args, **kwargs)

    def __deepcopy__(self, memo):
        import copy
        eng, self._engine = self._engine, None
        try:
            cls = self.__class__
            new = cls.__new__(cls)
            memo[id(self)] = new
            for k, v in self.__dict__.items():
                setattr(new, k, copy.deepcopy(v, memo))
        finally:
            self._engine = eng
        return new


# ------------------------------------------------------------------------------------------------
# presets and registrations
# ------------------------------------------------------------------------------------------------
_SIZE = {
    "s": dict(layer_blocks=[2, 2, 3, 2], layer_channels=[16, 24, 32, 64], attn_blocks=[1, 1, 1, 1],
              head_dims=[8, 8, 8, 16], msmc_kernel_sizes=[5, 7], mlp_ratio=2,
              path_drop_rate=0.1, attn_drop_rate=0.1, key_drop_rate=0.1, mlp_drop_rate=0.1, other_drop_rate=0.1),
    "m": dict(layer_blocks=[2, 3, 6, 2], layer_channels=[24, 32, 64, 96], attn_blocks=[1, 1, 1, 1],
              head_dims=[8, 8, 16, 32], msmc_kernel_sizes=[5, 7], mlp_ratio=2,
              path_drop_rate=0.1, attn_drop_rate=0.1, key_drop_rate=0.1, mlp_drop_rate=0.1, other_drop_rate=0.1),
    "l": dict(layer_blocks=[2, 3, 6, 3], layer_channels=[32, 32, 64, 128], attn_blocks=[1, 1, 2, 1],
              head_dims=[8, 8, 16, 32], msmc_kernel_sizes=[3, 5, 7, 11], mlp_ratio=3,
              path_drop_rate=0.2, attn_drop_rate=0.2, key_drop_rate=0.1, mlp_drop_rate=0.2, other_drop_rate=0.1),
}
_TASK = {
    "dpk": dict(head="dpk", head_out_channels=3, head_sigmoid=True),
    "pmp": dict(head="cls", head_num_classes=2),
    "emg": dict(head="reg", head_scale=8.0),
    "baz": dict(head="reg", head_scale=360.0),
    "dis": dict(head="reg", head_scale=500.0),
}
# per-variant drop-rate overrides (all five rates set to the value), reference :953-1034
_DROP_OVERRIDE = {"m_dpk": 0.2, "l_dpk": 0.3, "s_pmp": 0.2, "m_pmp": 0.25, "l_pmp": 0.3}


def _make_creator(size: str, task: str):
    name = f"seist_{size}_{task}"

    def creator(**kwargs):
        cfg = dict(_SIZE[size])
        cfg.update(_TASK[task])
        rate = _DROP_OVERRIDE.get(f"{size}_{task}")
        if rate is not None:
            explicit = ("path_drop_rate", "attn_drop_rate", "key_drop_rate", "mlp_drop_rate", "other_drop_rate")
            for k in explicit:
                if k in kwargs:   # the reference passes these explicitly, so a caller override collides
                    raise TypeError(f"{name}() got multiple values for keyword argument '{k}'")
                cfg[k] = rate
        cfg.update(kwargs)
        return SeismogramTransformer(HParams(), **cfg)

    creator.__name__ = name
    creator.__qualname__ = name
    creator.__doc__ = f"SeisT-{size.upper()} / {task} (reference models/seist.py:940-1170)."
    creator.__module__ = __name__
    return creator


for _size in ("s", "m", "l"):
    for _task in ("dpk", "pmp", "emg", "baz", "dis"):
        _fn = register_model(_make_creator(_size, _task))
        globals()[_fn.__name__] = _fn
