"""The op-by-op float64 check of test_gpu_ops_at_scale.py at windows longer than 8192 samples, and the module and the
streaming picker at 16384 against the unmodified reference.

The attention keys of a window of L samples number L / 64 at every stage (attn_aggr_ratios 8, 4, 2, 1), so up to 8192
samples every attention op has at most 128 keys: one chunk of csrc/attention.cu.  The code accepts windows up to 16384
(preprocess.MAX_SAMPLES, pick_phase, ContinuousAnnotator / EventCharacterizer `window=`), where:
  * 16384: 256 keys, two full chunks, two att_bwd_kv key blocks per head; the default dispatch sends fewer convs to the
    wgmma engine and more to convk / pw_fwd than at 8192;
  * 10000: 157 keys, a partial second chunk with Lk % 4 != 0 (the per-key dropout mask across the chunk boundary); no
    conv runs on the tensor cores, the generic conv.cu kernels take 123 forward and 123 data-gradient ops, and bww runs
    up to ~105 chunks per CTA.
The batches keep about the benchmark's N x L (4.2 M samples), so arenas and persistent-loop counts stay near its own:
  * seist_m_dpk, 256 x 16384, training: default dispatch, and SEIST_TCC=1;
  * seist_m_dpk, 419 x 10000, training with the model's registered drop rates;
  * the shipped seist_m_dpk checkpoint, eval, 256 x 16384 on event records: trained attention is peaked, where a wrong
    rescale of the online softmax shows most.
All are held to the unchanged CHAN_TOL.  On an NVIDIA H100 80GB HBM3 at 700 W the four GPU op-by-op tests take about
80 s together (16384: 14 s, with SEIST_TCC=1 50 s including its child process; 10000: 12 s; pretrained eval: 4 s).

tests/golden/reference_long_window.pt (make_golden_long_window.py) holds the reference's float64 eval output of the
shipped seist_m_dpk and seist_s_dpk on 8 records of 16384 samples: the module forward at 16384 meets the criterion
test_gpu_pretrained.py applies at 8192, and ContinuousAnnotator(window=16384) equals the module forward of its windows.
"""
import hashlib
import os

import numpy as np
import pytest
import torch

import test_gpu_ops_at_scale as S
from harness import model_drops
from oracle import golden as G
from oracle import pretrained as PT
from seist_b200 import _lib
from seist_b200.models import create_model
from test_gpu_ops_at_scale_variants import plan_families

LONG = ("seist_m_dpk", 256, 16384)
MID = ("seist_m_dpk", 419, 10000)
LONG_SEED = 20260401                         # the records of the pretrained op-by-op check
FIXTURE = os.path.join(G.GOLD, "reference_long_window.pt")    # tests/golden/make_golden_long_window.py
FIXTURE_MODELS = ("seist_m_dpk", "seist_s_dpk")


# ---- what these configurations reach (CPU) ---------------------------------------------------------------------------
def _attention_ops(name, length, drops=None):
    from seist_b200 import plan as P
    m = create_model(name, in_channels=3, in_samples=length)
    m.set_drop_rates(**(drops or S.ZERO_DROPS))
    pl = P.PlanBuilder(m, P.FlatState(m, torch.device("cpu")), 1, length, True).build()
    return [f for f in pl.fwd_ops if f.kind == _lib.ATT_FWD]


@pytest.mark.parametrize("length,lk", [(16384, 256), (10000, 157)])
def test_attention_crosses_key_chunks(length, lk):
    """Every attention op has more than one 128-key chunk; at 10000 the last is partial and Lk % 4 != 0, so dropout
    takes the per-key mask path across the boundary."""
    ops = _attention_ops(MID[0], length, model_drops(MID[0]))
    assert len(ops) == 4 and all(f.L_in == lk for f in ops), [(f.L_out, f.L_in) for f in ops]
    assert all(f.p_attn > 0 for f in ops)
    if length == 10000:
        assert all(f.L_in % 128 and f.L_in % 4 for f in ops)
    assert all(f.L_in <= 128 for f in _attention_ops(MID[0], 8192))


@pytest.mark.parametrize("cfg,tcc_all", [(LONG, False), (LONG, True), (MID, False)], ids=["16384", "16384-tcc", "10000"])
def test_loop_counts_of_long_windows(cfg, tcc_all):
    """More than one iteration of every persistent loop each configuration has, and the host mirror of the launch rules
    assigns exactly the ops the library assigns to each persistent family (default dispatch)."""
    name, n, length = cfg
    lc = S.loop_counts(name, n, length, True, tcc_all)
    fams = plan_families(name, length, True)
    for what, by_phase in S.LOOP_FAMILY.items():
        assert not lc[what] or max(S.counts(lc, what)) > 1, (what, lc[what])
        if tcc_all:
            continue
        mirror = {(ph, i) for ph, i, _, _ in lc[what]}
        lib = {(ph, i) for ph, fam in by_phase.items() for i, f in enumerate(fams[ph]) if f == fam}
        assert mirror == lib, (what, "mirror only", sorted(mirror - lib), "library only", sorted(lib - mirror))
    if length == 16384:
        assert lc["tcconv tiles/CTA"] and (tcc_all or {2, 4} <= set(S.counts(lc, "pw_fwd G")))
    else:
        assert not lc["tcconv tiles/CTA"] and max(S.counts(lc, "bww chunks/CTA")) > 100


def test_plan_families_of_long_windows():
    """Which families each length reaches: at 16384 both wgmma directions with fewer ops than at 8192; at 10000 no
    tensor-core op and the generic conv.cu kernels for most convolutions."""
    at = {length: plan_families(MID[0], length, True) for length in (8192, 10000, 16384)}
    count = lambda length, ph, fam: at[length][ph].count(fam)          # noqa: E731
    for ph, fam in (("fwd", "tcconv_fwd(wgmma+TMA)"), ("bwd", "tcconv_bwd_data(wgmma+TMA)")):
        assert 0 < count(16384, ph, fam) < count(8192, ph, fam), (fam, count(16384, ph, fam), count(8192, ph, fam))
        assert count(10000, ph, fam) == 0
    assert count(16384, "fwd", "convk_fwd(simt)") > count(8192, "fwd", "convk_fwd(simt)")
    assert count(16384, "fwd", "pw_fwd(simt)") > count(8192, "fwd", "pw_fwd(simt)")
    assert count(10000, "fwd", "conv_fwd(simt)") > 100 and count(10000, "bwd", "conv_bwd_data(simt)") > 100
    for length in (10000, 16384):
        for ph, fam in (("fwd", "att_fwd"), ("bwd", "att_bwd_q"), ("bwd", "att_bwd_kv")):
            assert count(length, ph, fam) == 4


# ---- the op-by-op runs -----------------------------------------------------------------------------------------------
def _ran(rep, *families):
    missing = [f for f in families if not any(fam == f for fam, _ in rep.worst)]
    assert not missing, ("no op of these families was checked", missing)


@pytest.mark.gpu
def test_training_ops_at_16384():
    _ran(S.check_at_scale(*LONG, True), "att_fwd", "att_bwd_q", "att_bwd_kv", "tcconv_fwd(wgmma+TMA)",
         "tcconv_bwd_data(wgmma+TMA)")


@pytest.mark.gpu
def test_training_ops_at_16384_on_tensor_cores():
    S.check_on_tensor_cores(*LONG, families=("tcconv_fwd", "tcconv_bwd", "att_fwd"))


@pytest.mark.gpu
def test_training_ops_at_10000_with_dropout():
    rep = S.check_at_scale(*MID, True, model_drops(MID[0]), (1 << 40) + 0x5EED)
    _ran(rep, "att_fwd p_attn", "att_bwd_q p_attn", "att_bwd_kv p_attn", "conv_fwd(simt) p_elem",
         "conv_bwd_data(simt) p_elem", "res_bwd p_alpha")


@pytest.mark.gpu
def test_pretrained_eval_ops_at_16384():
    name, n, length = LONG
    S.check_at_scale(name, n, length, False, state_dict=PT.pretrained_state_dict(name),
                     x=PT.dpk_records(n, LONG_SEED, length), label="pretrained")


# ---- end to end against the reference at 16384 ---------------------------------------------------------------------
def load_fixture():
    return torch.load(FIXTURE, weights_only=False)


def test_fixture_matches_the_checkpoints_and_inputs():
    """The fixture was made from the checkpoints of reference_pretrained.pt and from these inputs."""
    fx = load_fixture()
    assert fx["length"] == 16384 and fx["n"] == len(PT.KINDS) and fx["seed"] == PT.DPK_SEED
    x = PT.dpk_records(fx["n"], fx["seed"], fx["length"])
    assert fx["x_sha256"] == hashlib.sha256(x.numpy().tobytes()).hexdigest()
    for name in FIXTURE_MODELS:
        e = fx["eval"][name]
        assert e["sha256"] == PT.fixture()["eval"][f"{name}_diting"]["sha256"]
        assert e["y"]["shape"] == (fx["n"], 3, 16384)
        assert int(e["well_posed"].sum()) >= 8


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURE_MODELS)
def test_eval_at_16384_matches_reference_float64(name):
    """The captured eval plan of the module at 16384 samples: the bound of test_gpu_pretrained.py (K_DEV x the
    reference's own fp32 deviation + FLOOR x its max-abs, and 1e-3 of it), and the P / S arg max where well posed."""
    from test_gpu_pretrained import FLOOR, K_DEV
    fx = load_fixture()
    e = fx["eval"][name]
    y_ref = PT.unsample64(e["y"])
    m = create_model(name, in_channels=3, in_samples=fx["length"])
    m.load_state_dict(PT.pretrained_state_dict(name), strict=True)
    m.cuda().eval()
    with torch.no_grad():
        y = m(PT.dpk_records(fx["n"], fx["seed"], fx["length"]).cuda()).cpu()
    err = y_ref.err(y)
    print(f"\n{name} L=16384: err {err:.3e}, reference fp32 dev {e['dev']:.3e}, err / dev {err / e['dev']:.3f}, "
          f"rel {err / y_ref.absmax:.3e}")
    assert err <= 1e-3 * y_ref.absmax
    assert err <= K_DEV * e["dev"] + FLOOR * y_ref.absmax, (err, e["dev"])
    wp = e["well_posed"]
    assert torch.equal(y[:, 1:].argmax(-1)[wp], e["pick"][wp]), (y[:, 1:].argmax(-1), e["pick"], wp)


@pytest.mark.gpu
def test_annotate_at_16384_equals_module_forward():
    """ContinuousAnnotator(window=16384) on one fixture record longer than a window: its stacked probabilities equal
    the module forward of its windows (2e-6, as test_gpu_stream.py at 8192)."""
    from oracle import stream_ref as SR
    from seist_b200 import preprocess as PP
    from seist_b200 import stream as ST
    name, W, stride = "seist_m_dpk", 16384, 4096
    m = create_model(name, in_channels=3, in_samples=W)
    m.load_state_dict(PT.pretrained_state_dict(name), strict=True)
    m.cuda().eval()
    g = torch.Generator().manual_seed(PT.DPK_SEED)
    rec = PT.record("event", g, 2 * W + 1234)[0].float()[None].cuda()
    T = rec.shape[-1]
    ann = ST.ContinuousAnnotator(m, window=W, stride=stride, batch=3)
    probs = ann.annotate(rec)
    starts = ST.window_starts(T, W, stride)
    assert len(starts) > 3 and starts[-1] == T - W
    x = torch.stack([rec[0, :, a:a + W] for a in starts]).contiguous()
    PP.normalize_(x, "std")
    with torch.no_grad():
        y = m(x).cpu().numpy()
    want = SR.stack(y, 1, T, W, stride, "mean")
    err = np.abs(probs.cpu().numpy() - want).max()
    assert err <= 2e-6, err
