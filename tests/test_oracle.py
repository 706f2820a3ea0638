"""CPU: pins oracle/vpt_oracle.py against (a) the live reference where its checkout is present (oracle/refshim.py), otherwise
the reference outputs stored in tests/golden by oracle/make_golden.py, (b) the invariants of SURVEY.md section 4."""
import glob
import os

import pytest
import torch

import make_golden
import refshim
import vpt_oracle as O

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
GOLD = [os.path.join(GOLDEN, n + ".pt") for n in ("tiny_plain", "tiny_perturbed")]


def golden(name):
    return torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)


def seeded_weights(fx):
    """The weights of a fixture (oracle/make_golden.py): seeded values on the reference's state-dict schema stored with it."""
    return make_golden.seeded_state_dict(make_golden.template_from(fx["schema"]), fx["wseed"], fx.get("perturbed", False))


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p) for p in GOLD])
def test_oracle_matches_golden(path):
    """The oracle against the reference's outputs stored by oracle/make_golden.py (the live comparison where the reference is absent)."""
    fx = torch.load(path, weights_only=False)
    cfg = O.Cfg(**fx["policy_kwargs"])
    sd = seeded_weights(fx)
    st = O.initial_state(cfg, fx["B"])
    with torch.no_grad():
        for (img, first), ch in zip(make_golden.forward_inputs(fx["B"]), fx["chunks"]):
            (pd, v, _), st = O.agent_policy_forward(sd, cfg, img, first, st)
            # same torch ops in the same order as the reference -> bit exact on the same machine; 1e-5 across machines
            assert torch.allclose(pd["camera"], ch["camera"], rtol=1e-5, atol=1e-5)
            assert torch.allclose(pd["buttons"][..., make_golden.COLS], ch["buttons"], rtol=1e-5, atol=1e-5)
            assert torch.allclose(v, ch["vpred"], rtol=1e-5, atol=1e-5)
            for s, (m, k, vv) in zip(st, ch["state"]):
                assert torch.equal(s[0], m)
                assert torch.allclose(s[1][0], k, rtol=1e-5, atol=1e-6) and torch.allclose(s[1][1], vv, rtol=1e-5, atol=1e-6)
    torch.manual_seed(7)
    ac = O.sample(pd)
    if torch.equal(pd["camera"], fx["chunks"][-1]["camera"]):  # identical logits -> sampling must be bit exact
        assert torch.equal(ac["camera"], fx["sample"]["camera"]) and torch.equal(ac["buttons"], fx["sample"]["buttons"])
    assert torch.allclose(O.logprob(pd, fx["sample"]), fx["sample_logprob"], rtol=1e-5, atol=1e-5)


def test_golden_fixtures_exist():
    assert len(GOLD) >= 2


@pytest.mark.parametrize("pert", [False, True])
def test_oracle_matches_live_reference(pert):
    if not refshim.available():
        return test_oracle_matches_golden(GOLD[int(pert)])
    pkw = refshim.policy_kwargs("2x", **refshim.TINY)
    pol = refshim.make_reference_agent_policy(pkw)
    if pert:
        make_golden.perturb(pol)
    sd = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    cfg = O.Cfg(**pkw)
    B = 3
    g = torch.Generator().manual_seed(0)
    st_r, st_o = pol.initial_state(B), O.initial_state(cfg, B)
    for ci, T in enumerate([8, 8, 3, 8, 1]):
        img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
        first = torch.zeros(B, T, dtype=torch.bool)
        if ci == 3:
            first[1, 0] = True
        with torch.no_grad():
            (pd, v, _), st_r = pol({"img": img}, first, st_r)
            (pd2, v2, _), st_o = O.agent_policy_forward(sd, cfg, img, first, st_o)
        for k in pd:
            assert torch.equal(pd[k], pd2[k])
        assert torch.equal(v, v2)
        for a, b in zip(st_r, st_o):
            assert torch.equal(a[0], b[0]) and torch.equal(a[1][0], b[1][0]) and torch.equal(a[1][1], b[1][1])
    torch.manual_seed(7)
    a1 = pol.pi_head.sample(pd)
    torch.manual_seed(7)
    a2 = O.sample(pd2)
    assert all(torch.equal(a1[k], a2[k]) for k in a1)
    assert torch.equal(pol.pi_head.logprob(a1, pd), O.logprob(pd2, a2))


def test_oracle_matches_live_reference_128px():
    """One full-size 128x128 frame through the 1x-width CNN path with reduced transformer (config C1 shape); against the stored
    reference outputs (oracle/make_golden.py) where the reference is absent."""
    if not refshim.available():
        fx = golden("forward_128px")
        pkw = fx["policy_kwargs"]
        cfg = O.Cfg(**pkw)
        with torch.no_grad():
            (pd, v, _), _ = O.agent_policy_forward(seeded_weights(fx), cfg, make_golden.img_128px(), torch.zeros(1, 1, dtype=torch.bool),
                                                   O.initial_state(cfg, 1))
        for k in ("camera", "buttons"):
            assert torch.allclose(pd[k], fx[k], rtol=1e-5, atol=1e-5), k
        assert torch.allclose(v, fx["vpred"], rtol=1e-5, atol=1e-5)
        return
    pkw = refshim.policy_kwargs("1x", n_recurrence_layers=1)
    pol = refshim.make_reference_agent_policy(pkw)
    sd = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    cfg = O.Cfg(**pkw)
    img = torch.randint(0, 256, (1, 1, 128, 128, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(3))
    first = torch.zeros(1, 1, dtype=torch.bool)
    with torch.no_grad():
        (pd, v, _), _ = pol({"img": img}, first, pol.initial_state(1))
        (pd2, v2, _), _ = O.agent_policy_forward(sd, cfg, img, first, O.initial_state(cfg, 1))
    assert torch.equal(pd["buttons"], pd2["buttons"]) and torch.equal(pd["camera"], pd2["camera"]) and torch.equal(v, v2)


def _tiny():
    fx = torch.load(GOLD[0], weights_only=False)
    return seeded_weights(fx), O.Cfg(**fx["policy_kwargs"])


def test_chunk_size_invariance():
    """SURVEY.md section 4 (i): N frames fed as chunks of 1/4/8 give the same logits."""
    sd, cfg = _tiny()
    img = torch.randint(0, 256, (2, 16, 32, 32, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(5))
    outs = []
    with torch.no_grad():
        for cs in (1, 4, 8):
            st, acc = O.initial_state(cfg, 2), []
            for t0 in range(0, 16, cs):
                (pd, _, _), st = O.agent_policy_forward(sd, cfg, img[:, t0:t0 + cs], torch.zeros(2, cs, dtype=torch.bool), st)
                acc.append(pd["camera"])
            outs.append(torch.cat(acc, 1))
    assert torch.allclose(outs[0], outs[1], atol=2e-5) and torch.allclose(outs[0], outs[2], atol=2e-5)


def test_reset_equals_fresh():
    """SURVEY.md section 4 (ii): first[b,0]=True at a chunk start == a fresh initial_state for that row."""
    sd, cfg = _tiny()
    g = torch.Generator().manual_seed(6)
    a = torch.randint(0, 256, (2, 8, 32, 32, 3), dtype=torch.uint8, generator=g)
    b = torch.randint(0, 256, (2, 8, 32, 32, 3), dtype=torch.uint8, generator=g)
    with torch.no_grad():
        _, st = O.agent_policy_forward(sd, cfg, a, torch.zeros(2, 8, dtype=torch.bool), O.initial_state(cfg, 2))
        first = torch.zeros(2, 8, dtype=torch.bool)
        first[:, 0] = True
        (pd1, _, _), _ = O.agent_policy_forward(sd, cfg, b, first, st)
        (pd2, _, _), _ = O.agent_policy_forward(sd, cfg, b, torch.zeros(2, 8, dtype=torch.bool), O.initial_state(cfg, 2))
    assert torch.allclose(pd1["buttons"], pd2["buttons"], atol=2e-5)


def test_flop_model_matches_survey():
    for w, gf in (("1x", 3.8213), ("2x", 15.0973), ("3x", 33.8278)):
        assert abs(O.forward_flops_per_frame(O.Cfg(**O.widths(w))) / 1e9 - gf) < 1e-3


def _gradient_matches_golden():
    fx = golden("gradient")
    pkw = fx["policy_kwargs"]
    cfg = O.Cfg(**pkw)
    sd = seeded_weights(fx)
    st_o = O.initial_state(cfg, fx["B"])
    for (img, first, actions), ch in zip(make_golden.gradient_inputs(fx["B"]), fx["chunks"]):
        leaf = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
        (pd_o, _, _), st_o = O.agent_policy_forward(leaf, cfg, img, first, st_o)
        loss_o = -O.logprob(pd_o, actions).mean()
        loss_o.backward()
        st_o = [(m, (k.detach(), v.detach())) for (m, (k, v)) in st_o]
        assert torch.allclose(loss_o.detach(), ch["loss"], rtol=1e-6, atol=0)
        n_checked = 0
        for name, ref in ch["grads"].items():
            gr = leaf[name].grad
            if ref is None:
                assert gr is None, name  # value head: untouched by the BC loss in both
                continue
            gflat = gr.flatten()
            # fp32 sums in another order on another host: each sampled element within 1e-5 of the parameter's gradient norm
            # (measured: <= 1.8e-6 across 1 to 32 CPU threads)
            assert torch.allclose(gflat[make_golden.grad_sample_index(name, gflat.numel())], ref["sample"], rtol=1e-5, atol=1e-5 * ref["norm"].item()), name
            assert torch.allclose(gflat.norm(), ref["norm"], rtol=1e-5, atol=1e-8), name
            n_checked += 1
        assert n_checked > 80


def test_oracle_gradient_matches_live_reference_autograd():
    """The BC step's parity target is autograd through the oracle (tests/test_training.py); this pins that target itself: the
    gradient of the BC loss (behavioural_cloning.py:101-123: -log-prob of the demonstrated action, KV memory detached between
    chunks) through the unmodified reference equals the gradient through the oracle, parameter by parameter (against the stored
    reference loss and gradient samples, oracle/make_golden.py, where the reference is absent)."""
    if not refshim.available():
        return _gradient_matches_golden()
    pkw = refshim.policy_kwargs("2x", **refshim.TINY)
    pol = refshim.make_reference_agent_policy(pkw)
    make_golden.perturb(pol)
    pol.train()  # as behavioural_cloning.py leaves it (no dropout / batch-norm in these models: same function)
    sd = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    cfg = O.Cfg(**pkw)
    B, T = 2, 8
    g = torch.Generator().manual_seed(3)
    st_r, st_o = pol.initial_state(B), O.initial_state(cfg, B)
    for ci in range(2):
        img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
        first = torch.zeros(B, T, dtype=torch.bool)
        actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g)}
        for p in pol.parameters():
            p.grad = None
        (pd, _, _), st_r = pol({"img": img}, first, st_r)
        loss_r = -pol.pi_head.logprob(actions, pd).mean()
        loss_r.backward()
        st_r = [(m, (k.detach(), v.detach())) for (m, (k, v)) in st_r]  # tree_map(lambda x: x.detach(), ...) :111
        leaf = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
        (pd_o, _, _), st_o = O.agent_policy_forward(leaf, cfg, img, first, st_o)
        loss_o = -O.logprob(pd_o, actions).mean()
        loss_o.backward()
        st_o = [(m, (k.detach(), v.detach())) for (m, (k, v)) in st_o]
        assert torch.equal(loss_r.detach(), loss_o.detach())
        n_checked = 0
        for name, p in pol.named_parameters():
            if p.grad is None:
                assert leaf[name].grad is None, name  # value head: untouched by the BC loss in both
                continue
            assert torch.allclose(p.grad, leaf[name].grad, rtol=1e-5, atol=1e-8), name
            n_checked += 1
        assert n_checked > 80
