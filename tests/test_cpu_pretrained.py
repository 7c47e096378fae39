"""not-gpu: the trained checkpoints the reference ships (oracle/pretrained.py, staged by oracle/build_ref.py) and what
the unmodified reference computed with them (tests/golden/reference_pretrained.pt, make_golden_pretrained.py).

The trained weights sit in a numerical regime the seeded parameters of the other fixtures never reach: BatchNorm
running variances down to 3.5e-10 (eps-dominated channels, a BN gain of ~316 x gamma), |running_mean| / std up to 8.6,
attention score spreads up to 30, saturated sigmoid heads.  These tests pin the two restatements the device tests use
as their references in that regime: oracle/seist_ref.forward (the GPU tests of tests/test_gpu_pretrained.py compare the
module path with the fixture directly) and oracle/plan_interp (the reference of the op-by-op checks at production
shapes), so that kernel ~ interpreter ~ reference holds with the trained weights too.
"""
import pytest
import torch

from oracle import golden as G
from oracle import pretrained as PT
from oracle import seist_ref as R
from oracle.plan_interp import Interp
from seist_b200 import plan as P
from seist_b200.models import create_model

IDS = [f"{n}_{d}" for n, d in PT.CHECKPOINTS]


def test_staged_checkpoints_match_fixture():
    """All 18 checkpoints are staged, byte for byte the files the fixture was made with, in the layout of this
    project's models (load_state_dict strict)."""
    assert sorted(PT.fixture()["eval"]) == sorted(IDS)
    for name, dataset in PT.CHECKPOINTS:
        sd = PT.pretrained_state_dict(name, dataset)
        assert G.digest(G.layout(sd)) == PT.fixture()["eval"][f"{name}_{dataset}"]["layout_sha"], (name, dataset)
        m = create_model(name, in_channels=3, in_samples=PT.WINDOW)
        assert G.layout(m.state_dict()) == G.layout(sd), (name, dataset)
        m.load_state_dict(sd, strict=True)


def test_missing_or_different_checkpoint_raises(tmp_path, monkeypatch):
    """A run without the staged checkpoints fails with the staging instruction instead of skipping."""
    monkeypatch.setattr(PT, "DIR", str(tmp_path))
    with pytest.raises(RuntimeError, match="run oracle/build_ref.py where a reference checkout exists"):
        PT.pretrained_state_dict("seist_m_dpk")
    (tmp_path / "seist_m_dpk_diting.pth").write_bytes(b"not the checkpoint")
    with pytest.raises(RuntimeError, match="run oracle/build_ref.py where a reference checkout exists"):
        PT.pretrained_state_dict("seist_m_dpk")


def test_inputs_are_the_documented_events():
    """The seeded batches have the kinds oracle/pretrained.py describes: picker windows normalised per channel, a
    zeroed channel, an early P, an S past the window end; characterisation windows with P at anchor(8192, 0.3)."""
    x, tgt, phases = PT.dpk_windows()
    assert x.shape == (8, 3, PT.WINDOW) and x.dtype == torch.float32
    for i, kind in enumerate(PT.KINDS):
        p, s = phases[i]
        live = x[i].abs().amax(-1) > 0
        assert live.sum() == (2 if kind == "zero_channel" else 3), kind
        assert torch.allclose(x[i][live].std(-1, unbiased=False), torch.ones(int(live.sum())), atol=1e-4)
        if kind == "noise":
            assert p is None and tgt[i].abs().max() == 0
        else:
            assert 0 <= p < PT.WINDOW and int(tgt[i, 1].argmax()) == p
        if kind == "early_p":
            assert p < 100
        if kind == "late_s":
            assert s >= PT.WINDOW and tgt[i, 2].abs().max() == 0
    xe = PT.event_windows()
    assert xe.shape == (7, 3, PT.WINDOW)
    a = int(PT.WINDOW * PT.P_RATIO)
    early = PT.EVENT_KINDS.index("early_p")
    head = xe[early, :, :a - 100]                     # cut before the record start: zeros, then the mean removed
    assert (head == head[:, :1]).all() and xe[early, :, a:].std(-1).min() > 0.5


@pytest.mark.parametrize("ckpt", PT.CHECKPOINTS, ids=IDS)
def test_oracle_float64_forward_equals_reference(ckpt):
    """oracle/seist_ref.forward in float64 with the trained weights equals the reference module in float64."""
    name, dataset = ckpt
    e = PT.load_eval(name, dataset)
    sd = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in PT.pretrained_state_dict(name, dataset).items()}
    with torch.no_grad():
        y, _ = R.forward(sd, PT.inputs(name).double(), R.spec_for(name), training=False)
    assert tuple(y.shape) == e["y"].shape
    assert e["y"].err(y) <= 1e-12 * e["y"].absmax, (e["y"].err(y), e["y"].absmax)


# The interpreter computes every op in float64 but keeps the activations between ops in the plan's fp32 arena (the
# state the kernels start from under teacher forcing), so it sits one fp32 rounding per stored activation away from
# the float64 reference: below the reference's own fp32 forward, which also rounds inside every sum.
@pytest.mark.parametrize("name", ["seist_s_dpk", "seist_s_pmp"])
def test_plan_interpreter_float64_equals_reference(name):
    e = PT.load_eval(name)
    m = create_model(name, in_channels=3, in_samples=PT.WINDOW)
    m.load_state_dict(PT.pretrained_state_dict(name), strict=True)
    m.eval()
    x = PT.inputs(name)
    pl = P.PlanBuilder(m, P.FlatState(m, torch.device("cpu")), x.shape[0], PT.WINDOW, training=False).build()
    P.allocate(pl, False)
    y = Interp(pl, torch.float64).run_fwd(x)
    y = y if pl.y_out.L > 1 else y[:, :, 0]
    err = e["y"].err(y)
    print(f"{name}: interpreter - float64 reference {err:.3e}, reference fp32 - float64 {e['dev']:.3e}")
    assert err <= e["dev"], (err, e["dev"])
