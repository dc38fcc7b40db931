"""GPU: the RL rollout decorating scaffolds with attachment points -- the captured `GraphedGeneratorRL` against the
eager `GraphGeneratorRL` replaying the same actions (log-likelihoods and parameter gradients to
test_gpu_rl_graphed's tolerances), and the recomputing backward's probabilities against the rollout's, bit for bit."""
import copy

import pytest
import torch

from tests.test_gpu_rl_graphed import _loss, _run
from tests.test_gpu_scaffold_generation import _gdb13_constants, attachment_lists, gdb13_scaffolds
from tests.test_gpu_generation_layouts import _seeded_model

pytestmark = pytest.mark.gpu

N = 13


def _setup(B=96):
    from graphinvent_b200.graphed import GraphedGeneratorRL
    C = _gdb13_constants()
    agent, _ = _seeded_model("GGNN", C, 1)
    prior, _ = _seeded_model("GGNN", C, 2)
    sn, se = gdb13_scaffolds()
    att = attachment_lists(sn, seed=1)
    gen = GraphedGeneratorRL(agent, B, constants=C, scaffolds=(sn, se), attachment=att)
    for s in range(1, 9):
        U = torch.rand(2 * N, B, generator=torch.Generator("cuda").manual_seed(s), device="cuda")
        with torch.no_grad():
            if not isinstance(_run(lambda: gen.build_graphs(agent, prior, uniforms=U)), Exception):
                return C, agent, prior, gen, U, (sn, se), att
    pytest.skip("no finished rollout among the seeds tried")


def test_masked_rollout_backward_matches_eager_autograd():
    from graphinvent_b200.generation import GraphGeneratorRL
    C, agent, prior, gen, U, sc, att = _setup()
    B = gen.batch_size
    _, agent_ll, prior_ll, _ = gen.sample(agent, prior, uniforms=U)
    R = gen.rounds
    p_a, p_b, acts = gen.p_a[:R].clone(), gen.p_b[:R].clone(), gen.act_rec[:R].clone()
    ids = gen.generated_scaffolds.clone()
    _loss(agent_ll, prior_ll).backward()
    assert gen.backward_rounds == [R, R]
    assert torch.equal(gen.recomputed_p[0][:R], p_a) and torch.equal(gen.recomputed_p[1][:R], p_b)
    agent2, prior2 = copy.deepcopy(agent), copy.deepcopy(prior)
    agent2.zero_grad()
    prior2.zero_grad()
    eager = GraphGeneratorRL(agent2, B, constants=C, scaffolds=sc, attachment=att)
    agent2.entry_capacity = prior2.entry_capacity = gen.entry_capacity
    try:
        _, ll_a, ll_p, _ = eager.sample(agent2, prior2, replay=list(acts))
    finally:
        agent2.entry_capacity = prior2.entry_capacity = None
    assert eager.rounds == R and torch.equal(eager.generated_scaffolds, ids)
    for name in ("generated_nodes", "generated_edges", "generated_n_nodes", "properly_terminated"):
        assert torch.equal(getattr(gen, name), getattr(eager, name)), name
    assert torch.allclose(ll_a, agent_ll, rtol=1e-5, atol=1e-6) and torch.allclose(ll_p, prior_ll, rtol=1e-5, atol=1e-6)
    _loss(ll_a, ll_p).backward()
    for m, m2 in ((agent, agent2), (prior, prior2)):
        total = sum(p.grad.norm().item() ** 2 for p in m2.parameters()) ** 0.5
        for p, p2 in zip(m.parameters(), m2.parameters()):
            assert (p.grad - p2.grad).norm().item() <= 1e-4 * p2.grad.norm().item() + 1e-5 * total


def test_set_scaffolds_between_rollout_and_backward_raises():
    C, agent, prior, gen, U, (sn, se), att = _setup()
    _, agent_ll, prior_ll, _ = gen.sample(agent, prior, uniforms=U)
    gen.set_scaffolds((sn[::-1].copy(), se[::-1].copy()), att[::-1])
    with pytest.raises(RuntimeError, match="set_scaffolds was called between"):
        _loss(agent_ll, prior_ll).backward()
