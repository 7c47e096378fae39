"""Golden fixtures of the reference model (tests/golden/<model>.pt): what the unmodified reference computed for seeded
parameters and inputs.  TEST INFRASTRUCTURE ONLY.

A fixture stores digests of the reference checkpoint's layout (key, shape, dtype of every state_dict entry; parameter
order), the input sizes and the reference's results.  Parameters and inputs are regenerated here from seeds, so they
cost no storage; results are kept as a `Sample`: their values at seeded positions that always include the element of
largest magnitude, plus that magnitude.  `tests/golden/make_golden.py` writes the fixtures by running the reference
on exactly the tensors `load()` rebuilds.
"""
import hashlib
import os

import numpy as np
import torch

from oracle import seist_ref as R

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
FIXTURES = {  # model: (batch, length)
    "seist_s_dpk": (4, 8192),
    "seist_m_dpk": (2, 8192),
    "seist_m_emg": (2, 8192),
    "seist_s_pmp": (4, 8192),      # HeadClassification + CELoss(weight=[1, 1])
    "seist_s_baz": (4, 8192),      # HeadRegression x 360 + HuberLoss
}
X_SEED, TARGET_SEED, PARAM_SEED = 20240921, 5, 17


def layout(state_dict):
    """[(key, shape, dtype name)] of a state_dict."""
    return [(k, tuple(v.shape), str(v.dtype).replace("torch.", "")) for k, v in state_dict.items()]


def digest(items):
    return hashlib.sha256("\n".join(map(repr, items)).encode()).hexdigest()


def synth_state_dict(lay, seed=PARAM_SEED):
    """Non-degenerate parameters for a layout [(key, shape, dtype)]: weights N(0, 0.5^2 / fan-in), norm scales near 1,
    small biases, plausible running statistics (random-init eval output is a flat 0.5).  Larger weights make some
    gradients of the fixtures ill-conditioned: sums with so much cancellation that fp32 kernels which merely add in a
    different order miss the 2e-3 gradient tolerance."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for key, shape, dtype in lay:
        dt = getattr(torch, dtype)
        if not dt.is_floating_point:
            sd[key] = torch.zeros(shape, dtype=dt)
        elif key.endswith("running_var"):
            sd[key] = 0.5 + torch.rand(shape, generator=g)
        elif key.endswith("running_mean"):
            sd[key] = 0.1 * torch.randn(shape, generator=g)
        elif len(shape) > 1:
            sd[key] = 0.5 * torch.randn(shape, generator=g) / float(np.prod(shape[1:])) ** 0.5
        elif key.endswith("weight"):
            sd[key] = 1.0 + 0.05 * torch.randn(shape, generator=g)
        else:
            sd[key] = 0.2 * torch.randn(shape, generator=g)
    return sd


def model_state_dict(name, length, seed=PARAM_SEED):
    """Seeded parameters in the layout of this project's model `name` (equal to the reference checkpoint's layout)."""
    from seist_b200.models import create_model
    return synth_state_dict(layout(create_model(name, in_channels=3, in_samples=length).state_dict()), seed)


def synth_inputs(name, n, length):
    """(x, target) of a fixture: R.synth_waveforms, with class / regression targets for the non-dpk heads."""
    x, tgt = R.synth_waveforms(n, length, seed=X_SEED)
    if name.endswith("pmp"):
        cls = torch.randint(0, 2, (n,), generator=torch.Generator().manual_seed(TARGET_SEED))
        tgt = torch.nn.functional.one_hot(cls, 2).float()
    elif name.endswith("baz"):
        tgt = torch.rand(n, 1, generator=torch.Generator().manual_seed(TARGET_SEED)) * 360.0
    elif not name.endswith("dpk"):
        tgt = torch.rand(n, 1, generator=torch.Generator().manual_seed(TARGET_SEED)) * 8.0
    return x, tgt


class Sample:
    """A reference tensor kept at fixed flat positions (always including its largest magnitude) and its max |.|."""

    def __init__(self, shape, idx, val, absmax):
        self.shape, self.idx, self.val, self.absmax = tuple(shape), idx.long(), val, float(absmax)

    @staticmethod
    def positions(numel, k, seed, argmax):
        """Every element of a small tensor, else k seeded positions and the arg max of |t|."""
        if numel <= k:
            return torch.arange(numel)
        return torch.cat([torch.randperm(numel, generator=torch.Generator().manual_seed(seed))[:k], torch.tensor([argmax])])

    @staticmethod
    def take(t, k, seed):
        """Stored form of t: values at `positions`, arg max and max of |t| (the positions themselves are recomputed)."""
        flat = t.detach().reshape(-1).double()
        amax = int(flat.abs().argmax())
        return flat[Sample.positions(flat.numel(), k, seed, amax)].float(), amax, flat.abs().max().item()

    @staticmethod
    def stored(shape, k, seed, val, argmax, absmax):
        return Sample(shape, Sample.positions(int(np.prod(shape)), k, seed, argmax), val, absmax)

    @staticmethod
    def whole(t):
        """Every element of t."""
        t = t.detach().cpu()
        return Sample(t.shape, torch.arange(t.numel()), t.reshape(-1), t.abs().max().item())

    def err(self, t):
        """max |t - reference| over the stored positions; a t with fewer leading rows is compared on the rows it has."""
        flat = t.detach().cpu().reshape(-1)
        keep = self.idx < flat.numel()
        return (flat[self.idx[keep]].double() - self.val[keep].double()).abs().max().item()


def pack(tensors, k, seed=0):
    """Samples of the tensors of a list, in three flat arrays; unpack() needs the same shapes in the same order."""
    vals, amax, mx = [], [], []
    for i, t in enumerate(tensors):
        v, a, m = Sample.take(t, k, seed + i)
        vals.append(v)
        amax.append(a)
        mx.append(m)
    return {"k": k, "seed": seed, "val": torch.cat(vals), "argmax": torch.tensor(amax), "absmax": torch.tensor(mx, dtype=torch.float64)}


def unpack(p, shapes):
    out, o = [], 0
    assert len(shapes) == p["argmax"].numel()
    for i, shape in enumerate(shapes):
        n = int(np.prod(shape))
        c = n if n <= p["k"] else p["k"] + 1
        out.append(Sample.stored(shape, p["k"], p["seed"] + i, p["val"][o:o + c], int(p["argmax"][i]), float(p["absmax"][i])))
        o += c
    assert o == p["val"].numel()
    return out


def load(name):
    """The fixture of model `name` with its parameters and inputs rebuilt: state_dict, x, target, loss, y_eval /
    y_train (Sample), grads / buffers_after ({key: Sample}), layout_sha / param_sha (digests of the reference's
    state_dict layout and parameter order), and for the dpk heads: pick (eval arg max of the P / S rows), det_above /
    det_amb ((N, L) bool: eval detection row > 0.5, and within 2e-3 of 0.5)."""
    from seist_b200.models import create_model
    g = torch.load(os.path.join(GOLD, f"{name}.pt"))
    n, length = g["batch"], g["length"]
    out = dict(g)
    out["state_dict"] = model_state_dict(name, length)
    out["x"], out["target"] = synth_inputs(name, n, length)
    for k in ("y_eval", "y_train"):
        out[k] = unpack(g[k], [g["y_shape"]])[0]
    m = create_model(name, in_channels=3, in_samples=length)     # key order pinned by layout_sha / param_sha
    for k, named in (("grads", m.named_parameters()), ("buffers_after", m.named_buffers())):
        keys, shapes = zip(*[(key, tuple(t.shape)) for key, t in named])
        out[k] = dict(zip(keys, unpack(g[k], shapes)))
    for k in ("det_above", "det_amb"):
        if k in g:
            bits = np.unpackbits(g[k].numpy(), axis=-1)[:, :length]
            out[k] = torch.from_numpy(bits.astype(bool))
    return out
