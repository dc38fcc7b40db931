"""GPU: the RL rollout as captured rounds and its backward by recomputation (graphinvent_b200.graphed.GraphedGeneratorRL)
against the captured generator, the eager `generation.GraphGeneratorRL`, fp64 restatements of the new kernels and the
reference's RL trace."""
import copy
import ctypes
import os

import numpy as np
import pytest
import torch

from tests.conftest import GOLDEN, MODELS, pretrained_path
from tests.test_gpu_generation_graphed import STATE, _small, _uniforms

pytestmark = pytest.mark.gpu


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _pair(model, seeds=(0, 1)):
    C, agent = _small(model, seed=seeds[0])
    _, prior = _small(model, seed=seeds[1])
    return C, agent, prior


def _run(fn):
    try:
        return fn()
    except RuntimeError as e:
        return e


def _eager_replay(agent, prior, C, B, actions, capacity):
    """eager GraphGeneratorRL replaying `actions` [R, B] with both models in capacity mode at `capacity`"""
    from graphinvent_b200.generation import GraphGeneratorRL
    eager = GraphGeneratorRL(agent, B, constants=C)
    agent.entry_capacity = prior.entry_capacity = capacity
    try:
        out = eager.sample(agent, prior, replay=list(actions))
    finally:
        agent.entry_capacity = prior.entry_capacity = None
    return eager, out


def _softmax_gather64(logits, a):
    p = torch.softmax(logits.double(), dim=1)
    return p.gather(1, a.long().unsqueeze(1)).squeeze(1)


def _logits(model, nodes, edges, capacity):
    model.entry_capacity = capacity
    try:
        with torch.no_grad():
            return model(nodes.float(), edges.float())
    finally:
        model.entry_capacity = None


# ---- rollout ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", MODELS)
def test_rollout_equals_graphed_generator_and_eager_replay(model):
    from graphinvent_b200.graphed import GraphedGenerator, GraphedGeneratorRL
    C, agent, prior = _pair(model)
    B = 96
    U = _uniforms(C.max_n_nodes, B, 1)
    gen = GraphedGeneratorRL(agent, B, constants=C)
    with torch.no_grad():
        got = _run(lambda: gen.sample(agent, prior, uniforms=U))
    ref = GraphedGenerator(agent, B, constants=C)
    want = _run(lambda: ref.build_graphs(uniforms=U))
    assert type(got) is type(want) or not isinstance(want, Exception), (got, want)
    R = gen.rounds
    assert R == ref.rounds and gen.inert_rounds == 1
    for name in STATE:
        if name not in ("likelihoods", "generated_likelihoods"):   # RL rounds store slot tags there
            assert torch.equal(getattr(gen, name), getattr(ref, name)), name
    assert torch.equal(gen._counters, ref._counters)
    if isinstance(want, Exception):
        return
    acts = gen.act_rec[:R].clone()
    # the actions are the agent's draws; the probabilities are the softmax of the logits of the recorded input
    p_a, p_b = gen.p_a[:R].clone(), gen.p_b[:R].clone()
    for r in range(R):
        la = _logits(agent, gen.rec_nodes[r], gen.rec_edges[r], gen.entry_capacity)
        lb = _logits(prior, gen.rec_nodes[r], gen.rec_edges[r], gen.entry_capacity)
        for p, lg in ((p_a[r], la), (p_b[r], lb)):
            ref64 = _softmax_gather64(lg, acts[r])
            assert ((p.double() - ref64).abs() <= 4e-7 * ref64 + 1e-30).all(), r
    eager, out = _eager_replay(agent, prior, C, B, acts, gen.entry_capacity)
    assert eager.rounds == R
    for name in ("generated_nodes", "generated_edges", "generated_n_nodes", "properly_terminated"):
        assert torch.equal(getattr(gen, name), getattr(eager, name)), name
    for ours, theirs in ((gen.generated_agent_likelihoods, eager.generated_agent_likelihoods),
                         (gen.generated_prior_likelihoods, eager.generated_prior_likelihoods)):
        theirs = theirs.detach()
        assert torch.equal(ours != 0, theirs != 0)
        assert ((ours - theirs).abs() <= 4e-7 * theirs.abs()).all()
    assert torch.equal(got[3], out[3][:B])
    if model == "AttGGNN":
        # slot 0 samples two add actions with different bond types on the same bond: a multi-type bond the model
        # sees through the first-type view of the dummy graph, in the rollout and in the eager path alike
        acts2 = acts.clone()
        acts2[0, 0], acts2[1, 0] = 0, 1
        with torch.no_grad():
            gen.sample(agent, prior, actions=acts2)
        assert int((gen.edges[0] != 0).sum(-1).max()) == 2
        eager, _ = _eager_replay(agent, prior, C, B, acts2, gen.entry_capacity)
        assert torch.equal(gen.generated_edges, eager.generated_edges)
        assert ((gen.generated_agent_likelihoods - eager.generated_agent_likelihoods.detach()).abs()
                <= 4e-7 * eager.generated_agent_likelihoods.detach().abs()).all()


def test_reference_rl_trace_replayed_through_the_captured_rollout():
    path = pretrained_path()
    if path is None:
        pytest.skip("oracle/_ref/pretrained_model.pth absent: run __graft_entry__.build() with a checkout of the reference")
    from graphinvent_b200.config import make_constants
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.graphed import GraphedGeneratorRL
    from tests.test_zz_rl_rollout_gpu import _perturbed
    z = np.load(os.path.join(GOLDEN, "generation_rl_trace.npz"))
    B, n_gen, R = int(z["batch"]), int(z["n_generated"]), int(z["rounds"])
    sd = torch.load(path, map_location="cpu", weights_only=False)
    C = make_constants("GGNN")
    agent, prior = mpnn.create(C), mpnn.create(C)
    agent.load_state_dict(sd)
    prior.load_state_dict(_perturbed(sd, int(z["prior_seed"]), float(z["prior_noise"])))
    agent, prior = agent.cuda().train(), prior.cuda().eval()
    gen = GraphedGeneratorRL(agent, B, n_atom_types=5, n_formal_charge=3)
    _, agent_ll, prior_ll, _ = gen.sample(agent, prior, actions=torch.from_numpy(z["actions"]).cuda())
    assert gen.rounds == R and int(gen._counters[0]) == n_gen
    assert torch.equal(gen.generated_nodes.cpu().to(torch.int8), torch.from_numpy(z["generated_nodes"]))
    assert torch.equal(gen.generated_edges.cpu().to(torch.int8), torch.from_numpy(z["generated_edges"]))
    assert torch.equal(gen.generated_n_nodes.cpu(), torch.from_numpy(z["generated_n_nodes"]))
    assert torch.equal(gen.properly_terminated.cpu(), torch.from_numpy(z["properly_terminated"]))
    for ours, key in ((gen.generated_agent_likelihoods, "generated_agent_likelihoods"),
                      (gen.generated_prior_likelihoods, "generated_prior_likelihoods")):
        ref = torch.from_numpy(z[key])
        got = ours.detach().cpu()
        assert torch.equal(got != 0, ref != 0)
        rel = ((got - ref).abs() / ref.clamp(min=1e-12))[ref != 0]
        assert rel.max().item() <= 2e-2 and (rel <= 3e-4).float().mean().item() >= 0.85, (key, rel.max().item())
    assert (agent_ll.detach().cpu() - torch.from_numpy(z["agent_loglikelihoods"])).abs().max().item() <= 1e-2
    assert (prior_ll.detach().cpu() - torch.from_numpy(z["prior_loglikelihoods"])).abs().max().item() <= 1e-2
    assert (agent_ll.detach().cpu() - torch.from_numpy(z["agent_loglikelihoods"])).abs().median().item() <= 2e-4
    scores = torch.tensor([((i * 37) % 10) / 10.0 for i in range(B)], device="cuda")
    diff = agent_ll - (prior_ll + float(z["sigma"]) * scores)
    loss = torch.mean(diff * diff)
    assert abs(loss.item() - float(z["loss"])) <= 5e-3 * float(z["loss"])
    loss.backward()
    for tag, net in (("agent", agent), ("prior", prior)):
        names = [str(s) for s in z[f"grad_names_{tag}"]]
        ref_norm = dict(zip(names, z[f"grad_norm_{tag}"]))
        total = float(np.linalg.norm(z[f"grad_norm_{tag}"]))
        got_sq = 0.0
        for k, p in net.named_parameters():
            gn = p.grad.norm().item()
            got_sq += gn * gn
            assert abs(gn - ref_norm[k]) <= 5e-2 * ref_norm[k] + 1e-3 * total, (tag, k, gn, ref_norm[k])
        assert abs(got_sq ** 0.5 - total) <= 2e-2 * total


# ---- the backward kernels on their own -------------------------------------------------------------------------
@pytest.mark.parametrize("apd", [1, 2, 37, 625, 3361])
def test_rl_dlogits_against_fp64(apd):
    from graphinvent_b200._lib import check, lib
    g = torch.Generator().manual_seed(apd)
    B = 48
    logits = 4.0 * torch.randn(B, apd, generator=g)
    logits[3] *= 1e3                                     # saturated rows: most probabilities underflow to 0
    logits[4, :] = -1e4
    logits[4, apd // 2] = 1e4
    act = torch.randint(0, apd, (B,), generator=g, dtype=torch.int32)
    act[4] = apd // 2
    dp = torch.randn(B, generator=g)
    dp[::5] = 0.0                                        # rounds where a slot feeds no molecule
    dl = torch.full((B, apd), float("nan"), device="cuda")
    p = torch.full((B,), float("nan"), device="cuda")
    L, A, D = logits.cuda(), act.cuda(), dp.cuda()
    check(lib.gib_rl_dlogits(B, apd, _p(L), _p(A), _p(D), None, _p(dl), _p(p), _st()), "gib_rl_dlogits")
    s = torch.softmax(logits.double(), 1)
    p64 = s.gather(1, act.long().unsqueeze(1)).squeeze(1)
    onehot = torch.nn.functional.one_hot(act.long(), apd).double()
    ref = dp.double().unsqueeze(1) * p64.unsqueeze(1) * (onehot - s)
    # fp32 rounding: expf (2 ulp), the division, and the fp32 sum of exp over the row (relative ~1e-7 per level of
    # its 256-thread tree and per-thread strides); 1e-37: probabilities below fp32's normal range round to 0
    tol = 2e-6
    assert ((p.cpu().double() - p64).abs() <= tol * p64 + 1e-37).all(), ((p.cpu().double() - p64).abs() / p64).max()
    err = (dl.cpu().double() - ref).abs()
    assert (err <= 2 * tol * (dp.double().abs() * p64).unsqueeze(1) + 1e-37).all(), err.max().item()
    assert (dl.cpu()[::5] == 0).all()


def test_owner_map_gather_and_inversion_against_numpy():
    from graphinvent_b200._lib import check, lib
    rng = np.random.default_rng(3)
    B, Lw, rows = 40, 26, 80
    owner = np.zeros((rows, Lw), np.float32)
    for t in range(Lw):                              # each (round, slot) feeds at most one molecule; slot 0 none
        slots = rng.permutation(np.arange(1, B))[: rng.integers(0, B)]
        owner[rng.choice(rows, len(slots), replace=False), t] = slots + 1
    p_a, p_b = rng.random((Lw, B), np.float32), rng.random((Lw, B), np.float32)
    d_a, d_b = rng.standard_normal((rows, Lw)).astype(np.float32), rng.standard_normal((rows, Lw)).astype(np.float32)
    dev = [torch.from_numpy(x).cuda() for x in (owner, p_a, p_b, d_a, d_b)]
    out = [torch.full((rows, Lw), 7.0, device="cuda") for _ in range(2)]
    dp = [torch.full((Lw, B), 7.0, device="cuda") for _ in range(2)]
    check(lib.gib_rl_gather(B, rows, Lw, *map(_p, dev[:3] + out), _st()), "gib_rl_gather")
    check(lib.gib_rl_scatter_grad(B, rows, Lw, _p(dev[0]), _p(dev[3]), _p(dev[4]), _p(dp[0]), _p(dp[1]), _st()),
          "gib_rl_scatter_grad")
    want_out = [np.zeros((rows, Lw), np.float32) for _ in range(2)]
    want_dp = [np.zeros((Lw, B), np.float32) for _ in range(2)]
    for g in range(rows):
        for t in range(Lw):
            s = int(owner[g, t]) - 1
            if s >= 0:
                for k, (p, d) in enumerate(((p_a, d_a), (p_b, d_b))):
                    want_out[k][g, t] = p[t, s]
                    want_dp[k][t, s] = d[g, t]
    for k in range(2):
        assert (out[k].cpu().numpy() == want_out[k]).all()
        assert (dp[k].cpu().numpy() == want_dp[k]).all()
    assert (dp[0].cpu().numpy()[:, 0] == 0).all()


# ---- the backward through the whole rollout ------------------------------------------------------------------
def _loss(agent_ll, prior_ll):
    B = agent_ll.shape[0]
    w = torch.linspace(0.5, 1.5, B, device=agent_ll.device)
    return (w * agent_ll).sum() - (w.flip(0) * prior_ll).sum()


def _grads(model):
    return [p.grad.clone() if p.grad is not None else None for p in model.parameters()]


def _finished_rollout(model, B=96, seed=1):
    """models and uniforms whose rollout finishes within the round limit"""
    from graphinvent_b200.graphed import GraphedGeneratorRL
    C, agent, prior = _pair(model)
    for s in range(seed, seed + 8):
        U = _uniforms(C.max_n_nodes, B, s)
        gen = GraphedGeneratorRL(agent, B, constants=C)
        with torch.no_grad():
            if not isinstance(_run(lambda: gen.build_graphs(agent, prior, uniforms=U)), Exception):
                return C, agent, prior, gen, U
    pytest.skip("no finished rollout among the seeds tried")


@pytest.mark.parametrize("model", MODELS)
def test_backward_recomputes_the_rollout_and_matches_eager_autograd(model):
    C, agent, prior, gen, U = _finished_rollout(model)
    B = gen.batch_size
    _, agent_ll, prior_ll, _ = gen.sample(agent, prior, uniforms=U)
    R = gen.rounds
    p_a, p_b, acts = gen.p_a[:R].clone(), gen.p_b[:R].clone(), gen.act_rec[:R].clone()
    _loss(agent_ll, prior_ll).backward()
    assert gen.backward_rounds == [R, R]
    # the recomputed forward of every round gives the rollout's probabilities bit for bit
    assert torch.equal(gen.recomputed_p[0][:R], p_a) and torch.equal(gen.recomputed_p[1][:R], p_b)
    # the captured backward equals a host loop of the same C-ABI calls (the prior was the last model run: slot 1)
    got = torch.cat([g.reshape(-1) for g in _grads(prior)])
    b = gen._bwd
    b.gflat[1].zero_()
    b.ctl.zero_()
    for _ in range(R):
        gen._enqueue_backward_round(1)
    assert torch.equal(b.gflat[1], got)
    # eager autograd through the same rollout (ATen softmax-gather and autograd's sum over rounds)
    agent2, prior2 = copy.deepcopy(agent), copy.deepcopy(prior)
    agent2.zero_grad()
    prior2.zero_grad()
    eager, (_, ll_a, ll_p, _) = _eager_replay(agent2, prior2, C, B, acts, gen.entry_capacity)
    assert torch.allclose(ll_a, agent_ll, rtol=1e-5, atol=1e-6) and torch.allclose(ll_p, prior_ll, rtol=1e-5, atol=1e-6)
    _loss(ll_a, ll_p).backward()
    # dlogits differ from ATen's softmax backward by a few fp32 ulps (relative 1e-6); the model backward is
    # linear in them and the same kernels run in both paths, so the gradients agree to that order, up to the
    # conditioning of the sum over rounds
    for m, m2 in ((agent, agent2), (prior, prior2)):
        total = sum(p.grad.norm().item() ** 2 for p in m2.parameters()) ** 0.5
        for p, p2 in zip(m.parameters(), m2.parameters()):
            assert (p.grad - p2.grad).norm().item() <= 1e-4 * p2.grad.norm().item() + 1e-5 * total


def test_frozen_model_gets_no_gradient_and_no_backward():
    C, agent, prior, gen, U = _finished_rollout("GGNN")
    _, a_ll, p_ll, _ = gen.sample(agent, prior, uniforms=U)
    _loss(a_ll, p_ll).backward()
    both = _grads(agent)
    agent.zero_grad(set_to_none=True)
    prior.zero_grad(set_to_none=True)
    prior.requires_grad_(False)
    _, a_ll, p_ll, _ = gen.sample(agent, prior, uniforms=U)
    _loss(a_ll, p_ll).backward()
    assert gen.backward_rounds == [gen.rounds, 0]
    assert all(p.grad is None for p in prior.parameters())
    assert all(torch.equal(g, p.grad) for g, p in zip(both, agent.parameters()))
    agent.requires_grad_(False)
    _, a_ll, _, _ = gen.sample(agent, prior, uniforms=U)
    assert not a_ll.requires_grad


def test_learning_step_two_rollouts_one_backward():
    """Workflow.learning_step's shape: rollout (agent, prior) and rollout (BASF, agent) wait, then one backward"""
    from graphinvent_b200.optim import FlatAdam
    C, agent, prior, gen, U1 = _finished_rollout("GGNN", seed=1)
    basf = copy.deepcopy(agent)
    U2 = None
    for s in range(20, 28):
        U = _uniforms(C.max_n_nodes, gen.batch_size, s)
        with torch.no_grad():
            if not isinstance(_run(lambda: gen.build_graphs(basf, agent, uniforms=U)), Exception):
                U2 = U
                break
    if U2 is None:
        pytest.skip("no finished second rollout among the seeds tried")
    singles = []
    for (m1, m2), U in (((agent, prior), U1), ((basf, agent), U2)):
        for m in (agent, prior, basf):
            m.zero_grad(set_to_none=True)
        _, a, b, _ = gen.sample(m1, m2, uniforms=U)
        _loss(a, b).backward()
        singles.append(_grads(agent))
    for m in (agent, prior, basf):
        m.zero_grad(set_to_none=True)
    _, a1, b1, _ = gen.sample(agent, prior, uniforms=U1)
    _, a2, b2, _ = gen.sample(basf, agent, uniforms=U2)
    (_loss(a1, b1) + _loss(a2, b2)).backward()
    for p, g1, g2 in zip(agent.parameters(), *singles):
        assert torch.allclose(p.grad, g1 + g2, rtol=1e-6, atol=1e-9)
    # a parameter changed in place between a rollout and its backward
    _, a1, b1, _ = gen.sample(agent, prior, uniforms=U1)
    with torch.no_grad():
        next(prior.parameters()).add_(1e-3)
    with pytest.raises(RuntimeError, match="inplace"):
        _loss(a1, b1).backward()
    # after optimizer steps the next rollout runs the new weights: it equals a freshly built generator's
    from graphinvent_b200.graphed import GraphedGeneratorRL
    opt = FlatAdam(agent.parameters(), lr=1e-3)
    for _ in range(2):
        opt.zero_grad()
        _, a1, b1, _ = gen.sample(agent, prior, uniforms=U1)
        _loss(a1, b1).backward()
        opt.step()
    U3 = _uniforms(C.max_n_nodes, gen.batch_size, 40)
    with torch.no_grad():
        got = _run(lambda: gen.sample(agent, prior, uniforms=U3))
        fresh = GraphedGeneratorRL(agent, gen.batch_size, constants=C)
        want = _run(lambda: fresh.sample(agent, prior, uniforms=U3))
    assert type(got) is type(want)
    for name in STATE:
        assert torch.equal(getattr(gen, name), getattr(fresh, name)), name
    if not isinstance(want, Exception):
        assert torch.equal(gen.generated_agent_likelihoods, fresh.generated_agent_likelihoods)


def test_learning_step_memory_stays_within_the_size_queries():
    """B = 1000 at the reference's GGNN defaults: peak memory of two rollouts + one backward is the shared buffers
    plus two records, not one workspace per round and model"""
    import ctypes as ct
    from graphinvent_b200._lib import lib
    from graphinvent_b200.config import make_constants
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.graphed import GraphedGeneratorRL, rl_record_bytes
    C = make_constants("GGNN")
    torch.manual_seed(0)
    agent = mpnn.create(C).cuda()
    prior, basf = copy.deepcopy(agent).eval(), copy.deepcopy(agent)
    B = 1000
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    gen = GraphedGeneratorRL(agent, B, n_atom_types=5, n_formal_charge=3)
    g = torch.Generator(device="cuda").manual_seed(0)
    _, a1, b1, _ = gen.sample(agent, prior, generator=g)
    _, a2, b2, _ = gen.sample(basf, agent, generator=g)
    (_loss(a1, b1) + _loss(a2, b2)).backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    bd = ct.byref(gen.d)
    shared = (gen.workspace_bytes + lib.gib_model_bwd_scratch_bytes(bd, gen.hdr) + 2 * gen.packed[0].numel()
              + gen.cws.numel() + gen.gbuf.numel())
    record = rl_record_bytes(B, gen.N, gen.F, gen.Ef)
    state = 4 * (3 * B * gen.N * gen.N * gen.Ef + 3 * B * gen.N * gen.F)        # generation state + finished graphs
    slack = 256 << 20
    # the static record and the two rollouts' records
    assert peak <= shared + 3 * record + state + slack, (peak / 2**30, shared / 2**30, record / 2**20)
