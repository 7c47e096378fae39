"""Lane scheduler (seist_b200/schedule.py): every data dependence of the plan must be covered by stream order or by an
event edge.  Pure host logic: runs without a GPU."""
import os

import pytest
import torch

from seist_b200 import _lib, plan as P, schedule
from seist_b200.models import create_model


def _happens_before_ok(ops, c_ops, deps, n_lanes):
    """Replay the issue order with vector clocks: clock[l][m] = latest op of lane m known to be complete when lane l
    issues its next op.  A wait on the event recorded after op k (lane m) merges the clock lane m had at k."""
    clock = [[-1] * n_lanes for _ in range(n_lanes)]
    at_record = {}
    ev_op = {c_ops[i].rec_event: i for i in range(len(ops)) if c_ops[i].rec_event >= 0}
    lane_of = [c_ops[i].lane for i in range(len(ops))]
    for i in range(len(ops)):
        l = lane_of[i]
        for q in range(c_ops[i].n_wait):
            e = c_ops[i].wait_ev[q]
            assert e in ev_op, f"op {i} waits for an event nobody records"
            k = ev_op[e]
            assert k < i, f"op {i} waits for an event recorded later (op {k})"
            snap = at_record[k]
            clock[l] = [max(a, b) for a, b in zip(clock[l], snap)]
        for j in deps[i]:
            m = lane_of[j]
            if m == l:
                assert j < i
            else:
                assert clock[l][m] >= j, f"op {i} ({ops[i].name}, lane {l}) may run before its producer {j} ({ops[j].name}, lane {m})"
        clock[l][l] = i
        if c_ops[i].rec_event >= 0:
            at_record[i] = list(clock[l])
    return True


@pytest.mark.parametrize("n_main", [1, 2, 3])
@pytest.mark.parametrize("name", ["seist_s_dpk", "seist_m_dpk"])
def test_lane_schedule_covers_every_dependence(name, n_main):
    m = create_model(name, in_channels=3, in_samples=2048)
    flat = P.FlatState(m, torch.device("cpu"))
    pl = P.PlanBuilder(m, flat, 2, 2048, training=True).build()
    for ops in (pl.fwd_ops, pl.bwd_ops):
        c_ops = (_lib.SeistOp * len(ops))()
        info = schedule.schedule_lanes(pl, ops, c_ops, n_main=n_main)
        deps = schedule._deps(pl, ops)
        assert sum(info["ops_per_lane"]) == len(ops)
        assert all(0 <= c_ops[i].lane <= n_main for i in range(len(ops)))
        assert _happens_before_ok(ops, c_ops, deps, n_main + 1)
    # weight gradients stay off the main lanes except in the tail of the backward pass
    L = _lib
    ops = pl.bwd_ops
    c_ops = (_lib.SeistOp * len(ops))()
    schedule.schedule_lanes(pl, ops, c_ops, n_main=n_main)
    main_kinds = (L.CONV_BWD_DATA, L.RES_BWD, L.ATT_BWD_Q, L.ATT_BWD_KV, L.HEADVEC_BWD)
    last_main = max(i for i, o in enumerate(ops) if o.kind in main_kinds)
    for i, o in enumerate(ops):
        if o.kind == L.CONV_BWD_W and i < last_main:
            assert c_ops[i].lane == n_main


def test_plan_lane_count():
    m = create_model("seist_s_dpk", in_channels=3, in_samples=1024)
    flat = P.FlatState(m, torch.device("cpu"))
    assert P.PlanBuilder(m, flat, 2, 1024, training=True, world=1).build().n_main == 2
    assert P.PlanBuilder(m, flat, 2, 1024, training=True, world=2).build().n_main == 1


def test_data_parallel_plan_is_scheduled_per_segment_on_one_main_lane():
    """world = 2 without the peer-memory exchange: the plan is cut into segments with a statistic all-reduce between
    them, and seist_plan_run_lanes issues one segment per call, so each segment's schedule must stand on its own.  One
    main lane keeps every BN_PREPARE in plan order on every rank."""
    m = create_model("seist_s_dpk", in_channels=3, in_samples=2048)
    flat = P.FlatState(m, torch.device("cpu"))
    pl = P.finalize(P.PlanBuilder(m, flat, 2, 2048, training=True, world=2).build(), True)
    assert pl.n_main == 1
    for ops, c_ops, segs in ((pl.fwd_ops, pl.c_fwd, pl.fwd_segments), (pl.bwd_ops, pl.c_bwd, pl.bwd_segments)):
        assert len(segs) > 1
        for start, end, _ in segs:
            seg_ops, seg_c = ops[start:end], c_ops[start:end]
            assert _happens_before_ok(seg_ops, seg_c, schedule._deps(pl, seg_ops), pl.n_main + 1)
            n = end - start
            for c in seg_c:
                assert -1 <= c.rec_event < n
                assert all(0 <= c.wait_ev[q] < n for q in range(c.n_wait))
                if c.kind not in (_lib.CONV_BWD_W, _lib.STEM_COMPOSE_BWD):
                    assert c.lane == 0
