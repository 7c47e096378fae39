"""The trained SeisT checkpoints the reference ships (`pretrained/*.pth`) and seeded event inputs for them.  TEST
INFRASTRUCTURE ONLY.

The checkpoints are never committed.  `oracle/build_ref.py` copies them byte for byte into `oracle/_ref/pretrained/`,
and `pretrained_state_dict(name, dataset)` reads them only from there, after checking each file's SHA-256 against the one
tests/golden/reference_pretrained.pt recorded when the reference ran on it.  A missing or different file raises: a test
of the trained regime that cannot load its weights fails instead of passing without having run.

The inputs are event waveforms, not white noise: P and S bursts of seeded onset, frequency, decay and amplitude on a
noise floor (`record`), in five kinds (`KINDS`) - ordinary events, a noise-only trace, a trace with one zeroed channel
(as the drop-channel augmentation leaves it), a P within 100 samples of the window start and an S past the window end.
`dpk_windows` cuts the picker's input as `ContinuousAnnotator` does (the window at the record start, normalised "std");
`event_windows` cuts the characterisation models' input as `EventCharacterizer` does (P at `anchor(8192, 0.3)`,
normalised "std").  Both are regenerated from seeds; tests/golden/make_golden_pretrained.py stores what the reference
computed on them.
"""
import functools
import os

import numpy as np
import torch

from oracle import build_ref
from oracle import event_ref as ER
from oracle import golden as G
from oracle import preprocess_ref as PR

DIR = os.path.join(build_ref.OUT, "pretrained")
FIXTURE = os.path.join(G.GOLD, "reference_pretrained.pt")
HEADS = ("dpk", "pmp", "emg", "baz", "dis")
CHECKPOINTS = [(f"seist_{s}_{h}", "diting") for h in HEADS for s in "sml"] + \
              [(f"seist_{s}_emg", "pnw") for s in "sml"]             # the 18 files of the reference's pretrained/
STEP_MODELS = ("seist_s_dpk", "seist_m_dpk", "seist_l_dpk", "seist_m_pmp", "seist_m_emg")   # fine-tuning fixtures

WINDOW = 8192
RECORD = 2 * WINDOW
P_RATIO = 0.3                       # EventCharacterizer's p_position_ratio of the reference's demo
MODE = "std"                        # the normalisation of ContinuousAnnotator and EventCharacterizer
KINDS = ("event", "event", "event", "event", "noise", "zero_channel", "early_p", "late_s")
DPK_N, DPK_SEED = len(KINDS), 20260301          # the fixture's picker batch: one of each kind
EVENT_SEED = 20260302                            # the fixture's characterisation batch: the kinds with a P
THRESHOLD, MIN_PEAK_DIST, TOPKS = 0.3, 50, (1, 8)   # ContinuousAnnotator's ppk / spk default; 1 s at 50 Hz
LABEL_WIDTH, LABEL_SHAPE, CODA_RATIO = 20, "gaussian", 1.4


def sha256(path) -> str:
    return build_ref.sha256(path)


def checkpoint_path(name, dataset="diting") -> str:
    return os.path.join(DIR, f"{name}_{dataset}.pth")


def read_checkpoint(path):
    """The state dict of a checkpoint file (some are saved as {"model_dict": ...})."""
    blob = torch.load(path, map_location="cpu", weights_only=True)
    return dict(blob.get("model_dict", blob))


@functools.lru_cache(maxsize=1)
def fixture():
    return torch.load(FIXTURE, weights_only=False)


def pretrained_state_dict(name, dataset="diting"):
    """The trained parameters and BatchNorm statistics of checkpoint `<name>_<dataset>.pth`, read from the staged copy
    in oracle/_ref/pretrained/ and checked against the SHA-256 stored in the fixture."""
    key = f"{name}_{dataset}"
    want = fixture()["eval"][key]["sha256"]
    path = checkpoint_path(name, dataset)
    if not os.path.isfile(path):
        raise RuntimeError(f"checkpoint {key}.pth is not staged in {DIR}: "
                           "run oracle/build_ref.py where a reference checkout exists")
    if sha256(path) != want:
        raise RuntimeError(f"checkpoint {path} differs from the one the fixture was made with (SHA-256 {want}): "
                           "run oracle/build_ref.py where a reference checkout exists")
    return read_checkpoint(path)


# ---- seeded event inputs ---------------------------------------------------------------------------------------------
def record(kind, g, length=RECORD):
    """(3, length) float64 raw trace of one `kind` and its P and S samples (None where the trace has no event).  P lies
    in the first window (the picker's); "late_s" puts S past that window's end."""
    t = torch.arange(length, dtype=torch.float64)
    x = torch.randn(3, length, generator=g, dtype=torch.float64)
    if kind == "noise":
        return x, None, None
    u = lambda lo, hi: lo + (hi - lo) * float(torch.rand((), generator=g, dtype=torch.float64))   # noqa: E731
    if kind == "early_p":
        p = int(u(20, 100))
    elif kind == "late_s":
        p = int(u(6400, 7400))
    else:
        p = int(u(600, 4500))
    s = WINDOW + int(u(100, 1500)) if kind == "late_s" else p + int(u(150, 2500))
    amp = 10 ** u(0.3, 1.6)
    for onset, a, freq in ((p, amp, u(0.04, 0.16)), (s, amp * u(1.2, 3.0), u(0.015, 0.07))):
        decay = length / u(24, 96)
        env = torch.where(t >= onset, torch.exp(-(t - onset) / decay), torch.zeros((), dtype=torch.float64))
        ph = 2 * np.pi * torch.rand(3, 1, generator=g, dtype=torch.float64)
        gain = 0.4 + torch.rand(3, 1, generator=g, dtype=torch.float64)
        x += a * gain * env * torch.sin(2 * np.pi * freq * (t - onset) + ph)
    if kind == "zero_channel":
        x[int(torch.randint(0, 3, (1,), generator=g))] = 0.0
    return x, p, s


def _records(n, seed, kinds, length=RECORD):
    g = torch.Generator().manual_seed(seed)
    return [record(kinds[i % len(kinds)], g, length) for i in range(n)]


def dpk_windows(n=DPK_N, seed=DPK_SEED):
    """(x (n, 3, 8192) float32, target (n, 3, 8192) float32 [det, ppk, spk] labels, P / S samples): row i is of kind
    KINDS[i % 8], its first 8192 samples normalised as ContinuousAnnotator normalises a window."""
    xs, ts, phases = [], [], []
    for rec, p, s in _records(n, seed, KINDS):
        xs.append(PR.normalize(rec[:, :WINDOW].numpy().astype(np.float32), MODE))
        ps, ss = ([p], [s]) if p is not None else ([], [])
        ts.append(PR.dpk_labels(ps, ss, WINDOW, LABEL_WIDTH, LABEL_SHAPE, CODA_RATIO))
        phases.append((p, s))
    return torch.from_numpy(np.stack(xs)), torch.from_numpy(np.stack(ts)), phases


def dpk_records(n=DPK_N, seed=DPK_SEED, length=RECORD):
    """(n, 3, length) float32: the whole records of `dpk_windows` (row i of kind KINDS[i % 8]; the same records at the
    default length), each normalised "std" as one window of `length` samples."""
    return torch.from_numpy(np.stack([PR.normalize(rec.numpy().astype(np.float32), MODE)
                                      for rec, _, _ in _records(n, seed, KINDS, length)]))


EVENT_KINDS = tuple(k for k in KINDS if k != "noise")


def event_windows(n=len(EVENT_KINDS), seed=EVENT_SEED):
    """(n, 3, 8192) float32: row i an event of kind EVENT_KINDS[i % 7] cut from its record as EventCharacterizer cuts
    the window of a P pick (P at anchor(8192, 0.3), zero outside the record) and normalised "std"."""
    return torch.from_numpy(np.stack([ER.window(rec.numpy().astype(np.float32), p, WINDOW, P_RATIO, MODE)
                                      for rec, p, _ in _records(n, seed, EVENT_KINDS)]))


def inputs(name, n=None, seed=None):
    """The input batch of model `name`: dpk_windows for the pickers, event_windows for the other heads (the fixture's
    batch unless n / seed say otherwise)."""
    if name.endswith("dpk"):
        return dpk_windows(n or DPK_N, seed or DPK_SEED)[0]
    return event_windows(n or len(EVENT_KINDS), seed or EVENT_SEED)


def step_target(name, x):
    """The fine-tuning target of the fixture batch: dpk soft labels, pmp one-hot classes, emg magnitudes."""
    n = x.shape[0]
    if name.endswith("dpk"):
        return dpk_windows()[1]
    if name.endswith("pmp"):
        cls = torch.randint(0, 2, (n,), generator=torch.Generator().manual_seed(G.TARGET_SEED))
        return torch.nn.functional.one_hot(cls, 2).float()
    return torch.rand(n, 1, generator=torch.Generator().manual_seed(G.TARGET_SEED)) * 8.0


# ---- stored float64 results ------------------------------------------------------------------------------------------
def sample64(t, k, seed):
    """A float64 tensor kept at G.Sample's seeded positions (its largest magnitude included), values in float64."""
    flat = t.detach().reshape(-1).double()
    amax = int(flat.abs().argmax())
    return {"shape": tuple(t.shape), "k": k, "seed": seed, "argmax": amax, "absmax": flat.abs().max().item(),
            "val": flat[G.Sample.positions(flat.numel(), k, seed, amax)].clone()}


def unsample64(d):
    return G.Sample.stored(d["shape"], d["k"], d["seed"], d["val"], d["argmax"], d["absmax"])


def load_eval(name, dataset="diting"):
    """The fixture's eval entry of a checkpoint: sha256, layout_sha, y (G.Sample of the reference's float64 output),
    dev (max |fp32 - float64| of the reference's own forwards) and, for the pickers, pick / well_posed / det_above /
    det_amb / peaks / peaks_amb."""
    e = dict(fixture()["eval"][f"{name}_{dataset}"])
    e["y"] = unsample64(e["y"])
    for k in ("det_above", "det_amb"):
        if k in e:
            e[k] = torch.from_numpy(np.unpackbits(e[k].numpy(), axis=-1)[:, :WINDOW].astype(bool))
    return e


def load_step(name):
    """The fixture's fine-tuning step of checkpoint `<name>_diting`: x, target, loss, y_train (Sample), grads /
    buffers_after ({key: Sample})."""
    from seist_b200.models import create_model
    s = dict(fixture()["step"][name])
    s["x"] = inputs(name)
    s["target"] = step_target(name, s["x"])
    s["y_train"] = G.unpack(s["y_train"], [s["y_shape"]])[0]
    m = create_model(name, in_channels=3, in_samples=WINDOW)
    for k, named in (("grads", m.named_parameters()), ("buffers_after", m.named_buffers())):
        keys, shapes = zip(*[(key, tuple(t.shape)) for key, t in named])
        s[k] = dict(zip(keys, G.unpack(s[k], shapes)))
    return s
