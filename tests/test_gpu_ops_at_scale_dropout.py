"""The op-by-op float64 check of test_gpu_ops_at_scale.py with dropout on, as the benchmark trains: seist_m_dpk built
by `create_model` keeps its registered drop rates (stochastic depth spread over the blocks, attention-weight, key,
MLP and output-projection element dropout), and every kernel that applies a mask or a per-sample factor recomputes
the counter-based hash of csrc/common.cuh from its own (n, c, l) indices.

Dropout selects separate template instantiations (the `p_elem` bit of pw_fwd / pw_bwd_data / pw_bwd_data_staged, the
mask epilogues of tcconv, the quad and scalar attention masks), and its per-sample factors must follow each quad,
tile or chunk of a persistent loop across samples.  test_gpu_ops.py checks dropout at 2 x 1024 only, where every
persistent loop runs once; the configurations here run them many times:

  * the benchmark's step: (512, 3, 8192), default dispatch, and again with SEIST_TCC=1 (every eligible conv on the
    wgmma engine, many tiles per CTA, its forward and data-gradient mask code);
  * (500, 3, 6000): rows with L % 4 != 0 (the scalar keep_scale / elem_factor paths of the generic conv.cu kernels,
    res_bwd) and attention over Lk = 94 keys (the scalar mask path), with a step seed >= 2^63.

The CPU tests pin what these reach: the device masks of the interpreter equal its numpy ones bit for bit, no op
changes kernel family when dropout is on, each (family, dropout variant) of the plans is listed below and reached, and
the persistent loops of the dropout instantiations run more than one iteration.

Where a loop's iterations cross samples, a per-sample factor taken from the wrong iteration changes whole samples'
values, which the per-channel criterion catches (a pw_bwd_data_staged CTA that keeps the stochastic-depth factor of its
first tile fails the bench-shape test and passes test_gpu_ops.py).  The pw_fwd threads of the dropout ops do not cross
samples at the bench shape: the one such op with G > 1 has 256 quads per row, exactly G x 128, so each thread's quads
share a sample there.

The three GPU tests take about 70 s together on an NVIDIA H100 80GB HBM3 at 700 W, the CPU tests about a minute.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import test_gpu_ops_at_scale as S
from harness import ZERO_DROPS, model_drops
from oracle.plan_interp import keep_mask, keep_mask_range, keep_mask_t, rng_u16, rng_u16_t, rng_u64, rng_u64_t
from seist_b200 import _lib
from seist_b200 import plan as P
from seist_b200.models import create_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BENCH = (S.NAME, S.N, S.L)
RAGGED = ("seist_m_dpk", 500, 6000)
HIGH_SEED = (1 << 63) + 0x5EED          # a step counter with its top bit set: a negative value in the int64 tensor

# (kernel family, drop_label) of every dropout site of each plan: default dispatch / SEIST_TCC=1
_ATT = {("att_fwd", "p_attn"), ("att_bwd_q", "p_attn"), ("att_bwd_kv", "p_attn")}
_BWW = {("bww(simt)", "p_elem"), ("bww(simt)", "p_path")}
_TCC_FWD = {("tcconv_fwd(wgmma+TMA)", "p_elem"), ("tcconv_fwd(wgmma+TMA)", "p_path")}
_TCC_BWD = {("tcconv_bwd_data(wgmma+TMA)", "p_elem"), ("tcconv_bwd_data(wgmma+TMA)", "p_path")}
_PW = {("pw_fwd(simt)", "p_elem"), ("pw_fwd(simt)", "p_path"), ("pw_bwd_data(simt)", "p_elem"),
       ("pw_bwd_data(simt)", "p_path"), ("pw_bwd_data_staged(simt)", "p_elem")}
_CONV = {("conv_fwd(simt)", "p_elem"), ("conv_fwd(simt)", "p_path"), ("conv_bwd_data(simt)", "p_elem"),
         ("conv_bwd_data(simt)", "p_path"), ("res_bwd", "p_alpha")}
REACHED = {
    ("bench", False): _ATT | _BWW | _PW | {("pw_bwd_data_staged(simt)", "p_path"), ("res_bwd4", "p_alpha"),
                                           ("tcconv_fwd(wgmma+TMA)", "p_elem"), ("tcconv_fwd(wgmma+TMA)", "p_path")},
    ("bench", True): _ATT | _BWW | _TCC_FWD | _TCC_BWD | {("pw_bwd_data_staged(simt)", "p_elem"),
                                                          ("res_bwd4", "p_alpha")},
    ("ragged", False): _ATT | _BWW | _PW | _CONV | {("res_bwd4", "p_alpha"), ("tcconv_fwd(wgmma+TMA)", "p_elem")},
    ("ragged", True): _ATT | _BWW | _CONV | _TCC_FWD | _TCC_BWD | {("res_bwd4", "p_alpha")},
}
CFGS = {"bench": BENCH, "ragged": RAGGED}


# ---- the interpreter's device masks --------------------------------------------------------------------------------
def _as_int64(v):
    """A uint64 value as the int64 step_seed tensor stores it, read back as a Python int."""
    return int(torch.tensor([v - (1 << 64) if v >> 63 else v], dtype=torch.int64).item())


@pytest.mark.parametrize("p", [0.1, 0.2, 0.25])
def test_torch_masks_equal_numpy_masks(p):
    """rng_u64_t / rng_u16_t / keep_mask_t / keep_mask_range (int64 tensors, the interpreter's device masks) equal
    rng_u64 / rng_u16 / keep_mask (numpy uint64) bit for bit."""
    g = np.random.default_rng(5)
    idx = np.concatenate([g.integers(0, 1 << 40, 4096, dtype=np.uint64)] +
                         [np.arange(b - 64, b + 64, dtype=np.uint64) for b in (1 << 31, 1 << 32, 1 << 40)] +
                         [np.array([(1 << 62) + 3, (1 << 63) - 1, (1 << 63) + 2, (1 << 64) - 1], dtype=np.uint64)])
    assert set((idx & np.uint64(3)).tolist()) == {0, 1, 2, 3}
    tidx = torch.from_numpy(idx.view(np.int64))
    for seed in (0, 12345, (1 << 63) - 1, 1 << 63, HIGH_SEED, (1 << 64) - 1):
        s = _as_int64(seed)
        assert (s < 0) == (seed >= 1 << 63)
        for stream in (0, 7, (1 << 32) - 1):
            q = idx >> np.uint64(2)
            assert np.array_equal(rng_u64(s, stream, q).view(np.int64),
                                  rng_u64_t(s, stream, torch.from_numpy(q.view(np.int64))).numpy())
            assert np.array_equal(rng_u16(s, stream, idx).astype(np.int64), rng_u16_t(s, stream, tidx).numpy())
            ref = keep_mask(p, s, stream, idx)
            assert torch.equal(keep_mask_t(p, s, stream, tidx), ref)
            assert 0 < int((ref == 0).sum()) < len(idx)
            for n in (1, 6, 4099):
                assert torch.equal(keep_mask_range(p, s, stream, n, "cpu"),
                                   keep_mask(p, s, stream, np.arange(n, dtype=np.uint64)))
    # the signed and unsigned spellings of a seed draw the same masks
    assert torch.equal(keep_mask_t(p, _as_int64(HIGH_SEED), 3, tidx), keep_mask_t(p, HIGH_SEED, 3, tidx))


# ---- what the dropout configurations reach (CPU: the plan and the library's dispatch, no device) --------------------
def _plan(name, n, length, drops):
    m = create_model(name, in_channels=3, in_samples=length)
    m.set_drop_rates(**drops)
    return P.finalize(P.PlanBuilder(m, P.FlatState(m, torch.device("cpu")), n, length, True).build(), True)


def _families(name, length, drops, tcc_all):
    """seist_op_family of every op of a one-waveform training plan; with `tcc_all` in a child process with SEIST_TCC=1
    (the library reads it once per process)."""
    if not tcc_all:
        pl = _plan(name, 1, length, drops)
        return {"fwd": S._families(pl.c_fwd), "bwd": S._families(pl.c_bwd)}
    code = ("import sys, json; sys.path.insert(0, 'tests'); import test_gpu_ops_at_scale_dropout as T;"
            f"print('FAMILIES', json.dumps(T._families({name!r}, {length}, {drops!r}, False)))")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=dict(os.environ, SEIST_TCC="1"),
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.split("FAMILIES", 1)[1])


def _sites(pl, fams):
    """{(phase, op index): (family, drop_label)} of the plan's dropout sites."""
    out = {}
    for ph, i in S.dropout_sites(pl):
        op = (pl.fwd_ops if ph == "fwd" else pl.bwd_ops)[i]
        out[ph, i] = (fams[ph][i], S.drop_label(op.kind, op if ph == "fwd" else op.fwd))
    return out


def test_benchmark_model_trains_with_its_registered_drop_rates():
    """bench.py builds its model with create_model and never sets drop rates: the rates checked here are those."""
    drops = model_drops(S.NAME)
    assert all(v > 0 for v in drops.values()), drops
    assert drops == {k: getattr(create_model(S.NAME, in_channels=3, in_samples=S.L).hp, k) for k in ZERO_DROPS}


@pytest.mark.parametrize("cfg,tcc_all", [("bench", False), ("bench", True), ("ragged", False), ("ragged", True)],
                         ids=["bench", "bench-tcc", "ragged", "ragged-tcc"])
def test_dropout_sites_and_their_kernels(cfg, tcc_all):
    """Dropout moves no op to another kernel family (a pooled 1x1 conv with element dropout would leave pw_fwd, a
    k-tap one tcconv, but no op of these plans is either); every element mask sits on a 1x1 conv; the (family,
    variant) pairs of the dropout sites are those listed in REACHED, which the GPU tests must report; and the host
    mirror of the launch rules assigns exactly the library's ops to each persistent family."""
    name, n, length = CFGS[cfg]
    drops = model_drops(name)
    fams = _families(name, length, drops, tcc_all)
    assert fams == _families(name, length, ZERO_DROPS, tcc_all)
    pl = _plan(name, 1, length, drops)
    for f in pl.fwd_ops:
        if f.p_elem > 0:
            assert f.kind == _lib.CONV_FWD and f.k == 1 and f.pool <= 1 and f.up_src_L == 0, f.name
    sites = _sites(pl, fams)
    assert set(sites.values()) == REACHED[cfg, tcc_all], sorted(set(sites.values()) ^ REACHED[cfg, tcc_all])
    lc = S.loop_counts(name, n, length, True, tcc_all, drops)
    for what, by_phase in S.LOOP_FAMILY.items():
        mirror = {(ph, i) for ph, i, _, _ in lc[what]}
        lib = {(ph, i) for ph, fam in by_phase.items() for i, f in enumerate(fams[ph]) if f == fam}
        assert mirror == lib, (what, "mirror only", sorted(mirror - lib), "library only", sorted(lib - mirror))


@pytest.mark.parametrize("cfg", ["bench", "ragged"])
def test_dropout_sites_of_every_kind(cfg):
    """Each plan has forward and backward sites of every dropout kind; the attention masks take the quad path at the
    bench shape (Lk % 4 == 0) and the scalar one at the ragged length.  The GPU tests fail on any site that they do
    not hold to the per-channel criterion (check_at_scale), so a new site is covered or fails there."""
    name, n, length = CFGS[cfg]
    pl = _plan(name, n, length, model_drops(name))
    sites = S.dropout_sites(pl)
    labels = {}
    for ph, i in sites:
        op = (pl.fwd_ops if ph == "fwd" else pl.bwd_ops)[i]
        labels.setdefault(S.drop_label(op.kind, op if ph == "fwd" else op.fwd), set()).add(ph)
    assert labels == {"p_elem": {"fwd", "bwd"}, "p_path": {"fwd", "bwd"}, "p_alpha": {"bwd"}, "p_attn": {"fwd", "bwd"}}
    assert sum(f.p_alpha > 0 for f in pl.fwd_ops) > 0       # alpha scales the forward of its conv (label p_elem)
    print(f"\n{cfg}: {len(sites)} dropout sites, " + ", ".join(
        f"{k} {sum(getattr(f, k) > 0 for f in pl.fwd_ops)} fwd ops" for k in ("p_elem", "p_path", "p_alpha", "p_attn")))
    lks = {f.L_in for f in pl.fwd_ops if f.kind == _lib.ATT_FWD and f.p_attn > 0}
    assert lks and (all(lk % 4 == 0 for lk in lks) if cfg == "bench" else all(lk % 4 for lk in lks)), lks


def _bwd_data_loops(pl, fams, n):
    """(family, op index, iterations) of the pw_bwd_data / pw_bwd_data_staged ops with element dropout: quads per
    pw_bwd_data thread (pw.cu::pick_G) and a lower bound of the tiles per persistent pw_bwd_data_staged CTA (its grid is
    at most the resident CTAs: 32 per SM, or 2048 threads per SM / 32 per 16 input channels)."""
    out = []
    for i, (op, fam) in enumerate(zip(pl.bwd_ops, fams["bwd"])):
        f = op.fwd
        if op.kind != _lib.CONV_BWD_DATA or f.p_elem <= 0:
            continue
        if fam == "pw_bwd_data(simt)":
            cit = 16 if f.Cin > 8 else 8
            out.append((fam, i, S._pick_G(n * (f.L_out >> 2), -(-f.Cin // cit))))
        elif fam == "pw_bwd_data_staged(simt)":
            nt = 32 * -(-f.Cin // 16)
            out.append((fam, i, -(-n * (f.L_out >> 2) // 32) / (S.SM_COUNT * min(32, 2048 // nt))))
    return out


@pytest.mark.parametrize("cfg,tcc_all", [("bench", False), ("bench", True), ("ragged", False), ("ragged", True)],
                         ids=["bench", "bench-tcc", "ragged", "ragged-tcc"])
def test_dropout_instantiations_run_many_iterations(cfg, tcc_all):
    """At the bench shape each persistent family with an element-dropout op, and each with an op that has per-sample
    factors, runs more than one iteration of its loop on at least one of them (a thread / CTA crosses quads, tiles or
    chunks and so samples).  At the ragged length pw_fwd runs its dropout ops once per thread (500 x 47 quads are too
    few for G > 1), the other loops still run many times."""
    name, n, length = CFGS[cfg]
    drops = model_drops(name)
    pl = _plan(name, n, length, drops)
    lc = S.loop_counts(name, n, length, True, tcc_all, drops)
    ops = {"fwd": pl.fwd_ops, "bwd": [op.fwd for op in pl.bwd_ops]}
    for what in S.LOOP_FAMILY:
        if what == "pw_fwd G" and cfg != "bench":
            continue
        for kind, has in (("element mask", lambda f: f.p_elem > 0),
                          ("per-sample factor", lambda f: f.p_path > 0 or f.p_alpha > 0)):
            cs = [c for ph, i, _, c in lc[what] if has(ops[ph][i])]
            assert not cs or max(cs) > 1, (what, kind, cs)
    if cfg == "bench" and not tcc_all:
        assert max(c for ph, i, _, c in lc["pw_fwd G"] if ops[ph][i].p_elem > 0) > 1
    for what in ("tcconv tiles/CTA", "bww chunks/CTA"):
        assert max(c for ph, i, _, c in lc[what] if ops[ph][i].p_elem > 0) > 1, what
    if cfg == "bench" and not tcc_all:     # with SEIST_TCC=1 the wgmma engine takes most of these ops
        bd = _bwd_data_loops(pl, _families(name, length, drops, tcc_all), n)
        assert {f for f, _, _ in bd} == {"pw_bwd_data(simt)", "pw_bwd_data_staged(simt)"}, bd
        for fam in {f for f, _, _ in bd}:
            assert max(c for f, _, c in bd if f == fam) > 1, (fam, bd)


# ---- the op-by-op runs ------------------------------------------------------------------------------------------------
def _reached(rep, cfg, tcc_all):
    missing = [f"{fam} {label}" for fam, label in sorted(REACHED[cfg, tcc_all])
               if not any(k == f"{fam} {label}" for k, _ in rep.worst)]
    assert not missing, ("no op of these dropout variants was checked", missing)
    assert rep.sites and rep.sites <= rep.checked


@pytest.mark.gpu
def test_training_ops_at_bench_shape_with_dropout():
    """The benchmark's step: default drop rates and dispatch."""
    _reached(S.check_at_scale(*BENCH, True, model_drops(S.NAME)), "bench", False)


@pytest.mark.gpu
def test_training_ops_at_bench_shape_with_dropout_on_tensor_cores():
    """SEIST_TCC=1: the tcconv forward and data-gradient mask code, many tiles per CTA."""
    S.check_on_tensor_cores(*BENCH, families=tuple(f"{f} {lb}" for f, lb in sorted(REACHED["bench", True])),
                            drops=model_drops(S.NAME))


@pytest.mark.gpu
def test_training_ops_at_ragged_length_with_dropout():
    """Scalar mask paths (rows with L % 4 != 0, attention over Lk = 94 keys) and a step seed >= 2^63."""
    _reached(S.check_at_scale(*RAGGED, True, model_drops(RAGGED[0]), HIGH_SEED), "ragged", False)
