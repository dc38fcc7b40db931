"""GPU: the sampling policy (temperature / top-k / top-p, include/gib200.h `gib_sampling_policy`) -- the default is
today's sampler bit for bit, the kernel against the numpy restatement of tests/sampling_policy_reference.py on staged
and long rows, draws never leave the kept set, a chi-square test of the draw distribution, policy generation captured
equal to eager (masks and scaffolds included) with the model's likelihoods recorded, `set_sampling` without a
recapture, the RL rollout, guarded buffers and replay determinism."""
import copy
import ctypes

import numpy as np
import pytest
import torch

from tests import sampling_policy_reference as R
from tests.guarded import Guarded
from tests.test_gpu_action_mask import _check_batch, _gdb13_valence, _pretrained, _seeded_emn

pytestmark = pytest.mark.gpu

GRID_T = (0.0, 0.25, 0.7, 1.0, 1.5)
GRID_K = (0, 1, 5, 50)
GRID_P = (1.0, 0.9, 0.5, 1e-6)
GEN_STATE = ("generated_nodes", "generated_edges", "generated_n_nodes", "generated_likelihoods", "properly_terminated",
             "nodes", "edges", "n_nodes", "likelihoods")


def _rows(B, apd, seed):
    """logits [B, apd] fp32: N(0, 1) with ~20 % -inf; rows 0-3 all masked, one NaN, one +inf, one single finite entry;
    every 5th row rounded to 0.5 (exact ties, at the k-th place too)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, apd, generator=g, device="cuda")
    x[torch.rand(B, apd, generator=g, device="cuda") < 0.2] = -float("inf")
    x[::5] = torch.round(x[::5] * 2) / 2
    x[:, -1] = torch.randn(B, generator=g, device="cuda")           # terminate stays finite
    x[0] = -float("inf")
    x[1, apd // 2] = float("nan")
    x[2, 0] = float("inf")
    x[3] = -float("inf")
    x[3, apd // 3] = 0.5
    return x


def _sample(x, u, t, k, p):
    from graphinvent_b200 import functional as Fn
    return Fn.sample_actions(x, uniforms=u, temperature=t, top_k=k, top_p=p, return_policy=True)


# ---- 1. off is today ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("apd", [7, 625, 16411])
def test_off_policy_is_the_plain_sampler_bit_for_bit(apd):
    from graphinvent_b200 import functional as Fn
    x = _rows(4096, apd, 1)
    u = torch.rand(4096, generator=torch.Generator("cuda").manual_seed(2), device="cuda")
    a0, l0 = Fn.sample_actions(x, uniforms=u)
    a1, l1 = Fn.sample_actions(x, uniforms=u, temperature=1.0, top_k=0, top_p=1.0)
    a2, l2, q = Fn.sample_actions(x, uniforms=u, return_policy=True)        # the policy kernel with the policy off
    assert torch.equal(a0, a1) and torch.equal(l0.nan_to_num(7.0), l1.nan_to_num(7.0))
    assert torch.equal(a0, a2) and torch.equal(l0.nan_to_num(7.0), l2.nan_to_num(7.0))
    assert torch.equal(q[4:], l0[4:])                           # off: the policy's probability is the model's
    assert (a0[:3] == apd - 1).all() and l0[:3].isnan().all() and q[:3].isnan().all()


def test_default_graphed_generator_equals_one_built_without_a_policy():
    from graphinvent_b200.graphed import GraphedGenerator
    C, net = _pretrained()
    B = 256
    U = torch.rand(2 * 13, B, generator=torch.Generator("cuda").manual_seed(4), device="cuda")
    a = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3)
    b = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3, temperature=1.0, top_k=0, top_p=1.0)
    assert not b._policy_round and b.sampling == (1.0, 0, 1.0)
    a.build_graphs(uniforms=U)
    b.build_graphs(uniforms=U)
    for name in GEN_STATE:
        assert torch.equal(getattr(a, name), getattr(b, name)), name


# ---- 2. the kernel against the reference -------------------------------------------------------------------------
def _near(qr, u, tol=1e-5):
    """the entries whose inverse-CDF bracket lies within tol (relative) of the target u * total"""
    cdf = np.cumsum(qr)
    t = u * cdf[-1]
    lo = cdf - qr
    return set(np.flatnonzero((qr > 0) & (lo - tol * cdf[-1] <= t) & (t < cdf + tol * cdf[-1])).tolist())


@pytest.mark.parametrize("apd", [7, 625, 16411])
def test_kernel_matches_the_reference(apd):
    """the whole grid; every row is checked at apd 7 / 625, every 16th at 16411 (the long-row path).

    A draw whose uniform lies within 1e-5 (relative) of a CDF boundary must be one of the entries at that boundary.  A
    row whose kept set is decided within 2e-6 of the top-p threshold is skipped (its draw must still lie in the kept
    set at the larger threshold): the kernel's fp32 weights carry up to ~6e-7 relative error (the rounding of o - m
    and expf), so their running mass is that close to the fp64 one.  Skipped rows stay below 1 %.  The model's likelihood is checked to 2e-6 relative: fp32 rounding of o - m alone costs up to 5e-7
    at these logits, the fp32 expf and the chunked sum about as much again."""
    B = 4096
    x = _rows(B, apd, 3)
    xs = x.double().cpu().numpy()
    u = torch.rand(B, generator=torch.Generator("cuda").manual_seed(5), device="cuda")
    us = u.double().cpu().numpy()
    rows = range(B) if apd < 1000 else list(range(8)) + list(range(8, B, 16))
    checked = skipped = near = 0
    worst_lik = worst_q = 0.0
    for t in GRID_T:
        for k in GRID_K:
            for p in GRID_P:
                if t == 0 and (k, p) != (0, 1.0) and apd != 7:
                    continue                                    # greedy ignores k and p: covered at apd 7
                a, lik, q = (v.cpu().numpy() for v in _sample(x, u, t, k, p))
                for b in rows:
                    if R.degenerate(xs[b]):
                        assert a[b] == apd - 1 and np.isnan(lik[b]) and np.isnan(q[b]), (t, k, p, b)
                        continue
                    qr, kept, margin_p = R.policy(xs[b], t, k, p)
                    want, margin_u = R.draw(qr, us[b])
                    checked += 1
                    if margin_p < 2e-6:
                        skipped += 1
                        assert a[b] in R.policy(xs[b], t, k, min(1.0, p * (1 + 2e-6)))[1], (t, k, p, b)
                        continue
                    if margin_u < 1e-5:
                        near += 1
                        assert a[b] in _near(qr, us[b]), (t, k, p, b, a[b], want)
                    else:
                        assert a[b] == want, (t, k, p, b, a[b], want)
                    pm = R.model_prob(xs[b], a[b])
                    worst_lik = max(worst_lik, abs(lik[b] - pm) / pm)
                    worst_q = max(worst_q, abs(q[b] - qr[a[b]]) / qr[a[b]])
    print(f"apd {apd}: {checked} rows checked, {skipped} skipped at the top-p threshold, {near} near a CDF boundary")
    assert skipped <= 0.01 * checked, (skipped, checked)
    assert worst_lik <= 2e-6, worst_lik
    assert worst_q <= 2e-5, worst_q


# ---- 3. never outside the kept set -------------------------------------------------------------------------------
@pytest.mark.parametrize("apd", [625, 16411])
def test_draws_never_leave_the_kept_set(apd):
    rows, G = 6, 1001
    x = _rows(64, apd, 7)[[4, 5, 6, 10, 15, 20]]               # rows 10, 15, 20 have ties
    xs = x.double().cpu().numpy()
    xr = x.repeat_interleave(G, 0).contiguous()
    u = torch.linspace(0, 1, G + 1, device="cuda")[:-1].repeat(rows).contiguous()
    for t, k, p in ((0.7, 5, 0.9), (1.5, 0, 0.5), (0.25, 50, 1.0), (1.0, 1, 1.0), (0.0, 0, 1.0), (1.0, 0, 0.9)):
        a = _sample(xr, u, t, k, p)[0].view(rows, G).cpu().numpy()
        for r in range(rows):
            _, kept, margin_p = R.policy(xs[r], t, k, p)
            if margin_p < 1e-5:
                continue
            assert np.isin(a[r], kept).all(), (t, k, p, r, sorted(set(a[r]) - set(kept)))
            assert np.isfinite(xs[r][a[r]]).all()
            if t == 0 or k == 1:                                 # argmax, lowest index on ties
                assert (a[r] == R.ranking(xs[r])[0]).all()


# ---- 4. the draw distribution ------------------------------------------------------------------------------------
def test_two_hundred_thousand_draws_follow_the_policy():
    from scipy.stats import chisquare
    apd, n = 64, 200_000
    x = _rows(16, apd, 11)[6:7]
    t, k, p = 0.7, 20, 0.9
    qr, kept, _ = R.policy(x[0].double().cpu().numpy(), t, k, p)
    u = torch.rand(n, generator=torch.Generator("cuda").manual_seed(12), device="cuda")
    a = _sample(x.expand(n, apd).contiguous(), u, t, k, p)[0].cpu().numpy()
    assert np.isin(a, kept).all()
    obs = np.bincount(a, minlength=apd)[kept].astype(np.float64)
    exp = qr[kept] * n
    small = exp < 5                                             # pool the rare entries into one bin
    obs = np.append(obs[~small], obs[small].sum())
    exp = np.append(exp[~small], exp[small].sum())
    if exp[-1] == 0:
        obs, exp = obs[:-1], exp[:-1]
    assert len(kept) >= 5
    assert chisquare(obs, exp).pvalue > 1e-3


# ---- 5. generation -----------------------------------------------------------------------------------------------
def _eager_policy(model, C, B, U, pol, record=False, layout=(5, 3), **kw):
    """the eager generator's round loop on uniforms U [2N, B] with the policy, the model in capacity mode at the
    captured generator's capacity; record: per round (masked logits, action, likelihood, slot scaffold ids, atom
    counts), the last two None without scaffolds"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.generation import GraphGenerator
    from graphinvent_b200.graphed import entry_capacity, scaffold_entry_capacity
    lay = dict(n_atom_types=layout[0], n_formal_charge=layout[1]) if layout else {}
    gen = GraphGenerator(model, B, constants=C, **lay, **kw)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    model.entry_capacity = (entry_capacity(B, gen.N, gen.Ef) if gen.scaffolds is None else
                            scaffold_entry_capacity(B, gen.N, gen.Ef, gen.scaffolds.m_max))
    n, rnd, rec = 0, 0, []
    try:
        with torch.no_grad():
            while n < B:
                assert rnd < 2 * gen.N
                ids = gen._slot_ids.cpu().numpy() if record and gen.scaffolds is not None else None
                n_now = gen.n_nodes.cpu().numpy() if record else None
                out = model(*gen._model_inputs(model)).contiguous()
                if gen.masks_logits:
                    gen._mask(out, st)
                action, lik = Fn.sample_actions(out, uniforms=U[rnd], **pol._asdict())
                if record:
                    rec.append((out.double().cpu().numpy(), action.cpu().numpy(), lik.double().cpu().numpy(), ids,
                                n_now))
                gen._round(rnd, action, lik, st)
                n = int(gen._counters[0].item())
                rnd += 1
    finally:
        model.entry_capacity = None
    gen.rounds = rnd
    return gen, rec


# On the pretrained gdb13 GGNN, colder or narrower policies ((1, 0, 0.5), greedy, (0.7, 0, 0.9)) leave some slot
# running past the reference's 2N-round limit, where a batch raises in the eager and the captured generator alike;
# the seeded EMN finishes under all of them.
POLICIES = [("pretrained", (0.7, 0, 1.0)), ("pretrained", (1.3, 10, 0.9)), ("emn", (0.7, 0, 1.0)),
            ("emn", (1.3, 10, 0.9)), ("emn", (1.0, 0, 0.5)), ("emn", (0.0, 0, 1.0))]


@pytest.mark.parametrize("which,policy", POLICIES)
def test_policy_generation_captured_equals_eager_and_records_the_model(which, policy):
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.graphed import GraphedGenerator
    C, net = _pretrained() if which == "pretrained" else _seeded_emn()
    pol = Fn.sampling_policy(*policy)
    B = 256
    U = torch.rand(2 * C.max_n_nodes, B, generator=torch.Generator("cuda").manual_seed(21), device="cuda")
    gen = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3, **pol._asdict())
    assert gen._policy_round and gen.sampling == pol
    assert gen.build_graphs(uniforms=U) >= B
    eager, rec = _eager_policy(net, C, B, U, pol, record=True)
    assert eager.rounds == gen.rounds
    for name in GEN_STATE:
        assert torch.equal(getattr(gen, name), getattr(eager, name)), name
    worst = 0.0
    for logits, a, lik, _, _ in rec:
        for b in range(1, B, 3):
            if R.degenerate(logits[b]):
                continue
            pm = R.model_prob(logits[b], a[b])
            worst = max(worst, abs(lik[b] - pm) / pm)
            _, kept, margin_p = R.policy(logits[b], *pol)
            assert a[b] in kept or margin_p < 1e-5
    assert worst <= 2e-6, worst


@pytest.mark.parametrize("policy", [(1.3, 10, 0.9), (1.3, 10, 1.0)])
def test_policy_with_the_valence_mask_terminates_properly(policy):
    from graphinvent_b200.graphed import GraphedGenerator
    C, net = _pretrained()
    V = _gdb13_valence()
    B = 256
    gen = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3, action_mask="valence", max_valence=V,
                           temperature=policy[0], top_k=policy[1], top_p=policy[2])
    for seed in (1, 2):
        U = torch.rand(2 * 13, B, generator=torch.Generator("cuda").manual_seed(seed), device="cuda")
        assert gen.build_graphs(uniforms=U) >= B
        _check_batch(gen, B, "valence", V)
        if seed == 1:
            eager, _ = _eager_policy(net, C, B, U, gen.sampling, action_mask="valence", max_valence=V)
            for name in GEN_STATE:
                assert torch.equal(getattr(gen, name), getattr(eager, name)), name


def test_policy_with_scaffolds_and_attachment_points_draws_no_forbidden_action():
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.graphed import GraphedGenerator
    from tests import scaffold_oracle as SO
    from tests.test_gpu_generation_layouts import _seeded_model
    from tests.test_gpu_scaffold_generation import A, CH, EF, N, _forbidden, _gdb13_constants, attachment_lists, \
        gdb13_scaffolds
    sn, se = gdb13_scaffolds()
    att = attachment_lists(sn)
    C = _gdb13_constants()
    net, _ = _seeded_model("GGNN", C, 5)
    net.eval()
    B = 300
    pol = Fn.sampling_policy(1.3, 10, 0.9)
    U = torch.rand(2 * N, B, generator=torch.Generator("cuda").manual_seed(8), device="cuda")
    gen = GraphedGenerator(net, B, constants=C, scaffolds=(sn, se), attachment=att, **pol._asdict())
    gen.build_graphs(uniforms=U)
    eager, rec = _eager_policy(net, C, B, U, pol, record=True, layout=None, scaffolds=(sn, se), attachment=att)
    for name in GEN_STATE:
        assert torch.equal(getattr(gen, name), getattr(eager, name)), name
    k = eager.scaffolds.n_atoms
    protect = SO.protect_of(k, att, N)
    assert len(rec) == gen.rounds
    for logits, a, _, ids, n in rec:
        m = _forbidden(logits.shape, A * CH * EF, k, protect, ids, n)
        assert not m[np.arange(1, B), a[1:]].any()


# ---- 6. set_sampling without a recapture ---------------------------------------------------------------------------
def test_set_sampling_reuses_the_captured_round():
    from graphinvent_b200.graphed import GraphedGenerator
    C, net = _pretrained()
    B = 256
    U = torch.rand(2 * 13, B, generator=torch.Generator("cuda").manual_seed(9), device="cuda")
    gen = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3, temperature=1.3, top_k=10, top_p=0.9)
    gen.build_graphs(uniforms=U)
    graph = gen.graph
    for policy in ((1.3, 10, 1.0), (1.0, 0, 1.0), (0.7, 0, 1.0)):
        gen.set_sampling(*policy)
        gen.build_graphs(uniforms=U)
        assert gen.graph is graph
        fresh = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3, temperature=policy[0], top_k=policy[1],
                                 top_p=policy[2])
        fresh.build_graphs(uniforms=U)
        for name in GEN_STATE:
            assert torch.equal(getattr(gen, name), getattr(fresh, name)), (policy, name)
    # built without a policy: the first policy captures the round once, later ones reuse it
    plain = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3)
    plain.build_graphs(uniforms=U)
    g0 = plain.graph
    plain.set_sampling(1.3, 10, 0.9)
    plain.build_graphs(uniforms=U)
    g1 = plain.graph
    assert g1 is not g0
    plain.set_sampling(0.7)
    plain.build_graphs(uniforms=U)
    assert plain.graph is g1
    with pytest.raises(ValueError, match="top_p"):
        plain.set_sampling(top_p=0.0)


# ---- 7. RL -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mask", [None, "valence"])
def test_policy_rl_rollout_matches_eager(mask):
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.generation import GraphGeneratorRL
    from graphinvent_b200.graphed import GraphedGeneratorRL
    from tests.test_gpu_generation_layouts import _seeded_model
    from tests.test_gpu_rl_graphed import _loss
    C, agent = _pretrained()
    prior, _ = _seeded_model("GGNN", C, 2)
    V = _gdb13_valence() if mask else None
    B = 96
    pol = Fn.sampling_policy(1.3, 10, 0.9)
    gen = GraphedGeneratorRL(agent, B, n_atom_types=5, n_formal_charge=3, action_mask=mask, max_valence=V,
                             **pol._asdict())
    U = torch.rand(2 * 13, B, generator=torch.Generator("cuda").manual_seed(3), device="cuda")
    _, agent_ll, prior_ll, pt = gen.sample(agent, prior, uniforms=U)
    R_ = gen.rounds
    p_a, p_b, acts = gen.p_a[:R_].clone(), gen.p_b[:R_].clone(), gen.act_rec[:R_].clone()
    # every round's draw is the eager sampler's under the same policy and uniform, on the recorded state; p_a / p_b
    # are the models' probabilities of it
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    with torch.no_grad():
        for r in range(R_):
            xs, es = gen.rec_nodes[r].float(), gen.rec_edges[r].float()
            agent.entry_capacity = prior.entry_capacity = gen.entry_capacity
            try:
                la, lb = agent(xs, es).contiguous(), prior(xs, es).contiguous()
            finally:
                agent.entry_capacity = prior.entry_capacity = None
            if mask:
                for lg in (la, lb):
                    gen.action_mask.apply(B, lg, gen.rec_n[r], st, gen.rec_nodes[r], gen.rec_edges[r], int8=True)
            a, lik = Fn.sample_actions(la, uniforms=U[r], **pol._asdict())
            assert torch.equal(a, acts[r]), r
            assert torch.allclose(lik, p_a[r], rtol=1e-5, atol=0), r        # the agent's softmax at the draw
    agent.zero_grad()
    prior.zero_grad()
    _loss(agent_ll, prior_ll).backward()
    assert gen.backward_rounds == [R_, R_]
    assert torch.equal(gen.recomputed_p[0][:R_], p_a) and torch.equal(gen.recomputed_p[1][:R_], p_b)
    agent2, prior2 = copy.deepcopy(agent), copy.deepcopy(prior)
    agent2.zero_grad()
    prior2.zero_grad()
    eager = GraphGeneratorRL(agent2, B, n_atom_types=5, n_formal_charge=3, action_mask=mask, max_valence=V,
                             **pol._asdict())
    agent2.entry_capacity = prior2.entry_capacity = gen.entry_capacity
    try:
        _, ll_a, ll_p, _ = eager.sample(agent2, prior2, replay=list(acts))
    finally:
        agent2.entry_capacity = prior2.entry_capacity = None
    assert eager.rounds == R_
    for name in ("generated_nodes", "generated_edges", "generated_n_nodes", "properly_terminated"):
        assert torch.equal(getattr(gen, name), getattr(eager, name)), name
    assert torch.allclose(ll_a, agent_ll, rtol=1e-5, atol=1e-6) and torch.allclose(ll_p, prior_ll, rtol=1e-5, atol=1e-6)
    _loss(ll_a, ll_p).backward()
    for m, m2 in ((agent, agent2), (prior, prior2)):
        total = sum(p.grad.norm().item() ** 2 for p in m2.parameters()) ** 0.5
        assert total > 0
        for p, p2 in zip(m.parameters(), m2.parameters()):
            assert (p.grad - p2.grad).norm().item() <= 1e-4 * p2.grad.norm().item() + 1e-5 * total


# ---- 8. buffers ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("apd", [625, 16411])
def test_policy_kernel_stays_inside_its_buffers(apd):
    from graphinvent_b200._lib import check, lib
    B = 257
    x = _rows(B, apd, 13)
    u = torch.rand(B, generator=torch.Generator("cuda").manual_seed(14), device="cuda")
    gx, gu = Guarded.like(x), Guarded.like(u)
    pol = Guarded(16, fill="zero")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    check(lib.gib_sampling_policy_set(ctypes.c_void_p(pol.ptr()), 0.7, 5, 0.9, st), "gib_sampling_policy_set")
    outs = [Guarded(4 * B) for _ in range(3)]
    before = [g.raw.clone() for g in (gx, gu, pol)]
    check(lib.gib_sample_actions_policy(ctypes.c_void_p(gx.ptr()), B, apd, ctypes.c_void_p(gu.ptr()),
                                        ctypes.c_void_p(pol.ptr()), *(ctypes.c_void_p(g.ptr()) for g in outs), st),
          "gib_sample_actions_policy")
    torch.cuda.synchronize()
    for g, b0 in zip((gx, gu, pol), before):
        assert torch.equal(g.raw, b0)                            # inputs and their bands untouched
    for g in outs:
        assert g.intact(), g.damage()
    a = outs[0].view(torch.int32, (B,))
    assert ((a >= 0) & (a < apd)).all()
    a2, lik, q = _sample(x, u, 0.7, 5, 0.9)
    assert torch.equal(a, a2)
    for g, want in zip(outs[1:], (lik, q)):
        assert torch.equal(g.view(torch.float32, (B,)).nan_to_num(3.0), want.nan_to_num(3.0))


# ---- 9. determinism ----------------------------------------------------------------------------------------------
def test_replays_and_launches_are_deterministic():
    from graphinvent_b200.graphed import GraphedGenerator
    x = _rows(1024, 16411, 17)
    u = torch.rand(1024, generator=torch.Generator("cuda").manual_seed(18), device="cuda")
    first = _sample(x, u, 1.3, 50, 0.9)
    for _ in range(2):
        for v, w in zip(_sample(x, u, 1.3, 50, 0.9), first):
            assert torch.equal(v.nan_to_num(3.0), w.nan_to_num(3.0))
    C, net = _seeded_emn()
    B = 256
    U = torch.rand(2 * 13, B, generator=torch.Generator("cuda").manual_seed(19), device="cuda")
    gen = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3, temperature=0.7, top_k=10, top_p=0.9)
    gen.build_graphs(uniforms=U)
    keep = {name: getattr(gen, name).clone() for name in GEN_STATE}
    gen.build_graphs(uniforms=U)
    for name in GEN_STATE:
        assert torch.equal(getattr(gen, name), keep[name]), name
