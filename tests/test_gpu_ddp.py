"""-m gpu (needs >= 2 GPUs, skipped otherwise): two NCCL ranks running the fused train step with SyncBatchNorm
statistics exchanged at the plan's sync points must equal one rank on the concatenated batch (SURVEY §4.3)."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ZERO = dict(path_drop_rate=0, attn_drop_rate=0, key_drop_rate=0, mlp_drop_rate=0, other_drop_rate=0)
NAME, L, NB = "seist_s_dpk", 2048, 8


def _setup_model():
    from harness import randomize
    from seist_b200.models import create_model
    m = randomize(create_model(NAME, in_channels=3, in_samples=L), seed=5)
    m.set_drop_rates(**ZERO)
    return m


def _step(model, x, t, steps=1, use_graph=False):
    from seist_b200.train import Trainer
    # tiny learning rate: Adam's sign-like update would otherwise amplify last-bit gradient differences between the two
    # runs into the second (graph-replayed) step
    tr = Trainer(model, lr=1e-6, use_graph=use_graph)
    losses = [float(tr.step(x, t).item()) for _ in range(steps)]
    torch.cuda.synchronize()
    return losses, tr


def _worker(rank, world, port, q, use_graph, symm):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), SEIST_SYMM="1" if symm else "0")
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from oracle import seist_ref as R
    x, t = R.synth_waveforms(NB, L, seed=3)
    m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(_setup_model().cuda())
    n = NB // world
    losses, tr = _step(m, x[rank * n:(rank + 1) * n].cuda(), t[rank * n:(rank + 1) * n].cuda(), steps=2 if use_graph else 1,
                       use_graph=use_graph)
    assert (tr.plan.comm is not None) == symm
    if symm:
        assert not tr.plan.comm.timed_out(), "peer wait timed out"
        assert (tr.graph is not None) == use_graph
    lt = torch.tensor(losses[:1], device="cuda")
    dist.all_reduce(lt)
    if rank == 0:
        q.put(((lt / world).cpu(), (tr.last_grads / world).cpu().clone(), tr.flat.RB.cpu().clone()))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph,symm", [(False, True), (True, True), (False, False)],
                         ids=["peer-memory-eager", "peer-memory-graph", "nccl-fallback"])
def test_two_gpu_step_equals_single_gpu_on_concatenated_batch(use_graph, symm):
    """peer-memory: SyncBatchNorm statistics and gradients exchanged by the kernels themselves over NVLink symmetric
    memory (comm.cu) - eagerly and as ONE captured CUDA graph per rank (two steps: capture + replay; the first step is
    compared); nccl-fallback: SEIST_SYMM=0, NCCL calls at the plan's sync points."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q, use_graph, symm)) for r in range(2)]
    for p in procs:
        p.start()
    loss2, P2, RB2 = q.get(timeout=600)
    for p in procs:
        p.join(timeout=600)
        assert p.exitcode == 0
    from oracle import seist_ref as R
    x, t = R.synth_waveforms(NB, L, seed=3)
    losses, tr = _step(_setup_model().cuda(), x.cuda(), t.cuda(), steps=2 if use_graph else 1, use_graph=use_graph)
    losses = losses[:1]
    assert torch.allclose(loss2, torch.tensor(losses), rtol=1e-4, atol=1e-6), (loss2, losses)
    G1 = tr.last_grads.cpu()          # averaged gradient of the step (Adam normalises, so compare gradients, not weights)
    assert (P2 - G1).abs().max().item() < 2e-4 * G1.abs().max().item(), (P2 - G1).abs().max().item()
    assert (RB2 - tr.flat.RB.cpu()).abs().max().item() < 1e-3 * (tr.flat.RB.abs().max().item() + 1e-3)
