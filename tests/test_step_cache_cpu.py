"""The first-block step cache without a GPU: the skip policy on scripted changes, and the fp32 oracle of the rule
(tests/step_cache_ref.py) against the plain oracle and against itself replaying its own decisions."""
import math

import pytest
import torch

from diffusionkit_b200.step_cache import StepCachePolicy, max_relative_change


def _run(policy, rels):
    return [policy.decide(r) for r in rels]


def test_first_forward_after_reset_is_full():
    p = StepCachePolicy(math.inf)
    assert p.needs_full
    assert _run(p, [0.0, 0.0, 0.0]) == [False, True, True]
    assert p.log[0] == (None, False) and p.log[1] == (0.0, True)
    p.reset()
    assert p.needs_full and p.log == []
    assert _run(p, [0.0, 0.0]) == [False, True]


def test_threshold_edges():
    p = StepCachePolicy(0.1)
    assert _run(p, [None, 0.1, 0.0999999, 0.2, math.nextafter(0.1, 0.0)]) == [False, False, True, False, True]
    p = StepCachePolicy(0.0)                               # never skips, not even an unchanged residual
    assert _run(p, [None, 0.0, 0.0, 0.0]) == [False] * 4


@pytest.mark.parametrize("cap,want", [(None, "FSSSSS"), (0, "FFFFFF"), (1, "FSFSFS"), (2, "FSSFSS"), (3, "FSSSFS")])
def test_consecutive_cap(cap, want):
    p = StepCachePolicy(math.inf, cap)
    assert "".join("S" if s else "F" for s in _run(p, [0.0] * 6)) == want


def test_cap_counts_only_consecutive_skips():
    p = StepCachePolicy(0.5, 2)
    assert _run(p, [None, 0.1, 0.9, 0.1, 0.1, 0.1, 0.1]) == [False, True, False, True, True, False, True]


def test_zero_denominator_and_non_finite_never_skip():
    assert max_relative_change([(1.0, 2.0), (3.0, 4.0)]) == 0.75
    assert max_relative_change([(0.0, 0.0)]) == math.inf
    assert math.isnan(max_relative_change([(math.nan, 1.0)]))
    assert math.isnan(max_relative_change([(1.0, math.inf)]))
    p = StepCachePolicy(math.inf)
    assert p.step([(5.0, 1.0)]) is False                    # first forward: the sums are not looked at
    assert p.step([(0.0, 0.0)]) is False                    # zero denominator, even at threshold inf
    assert p.step([(0.0, 1.0), (0.0, 0.0)]) is False        # one sequence is enough to run the batch in full
    assert p.step([(math.nan, 1.0)]) is False
    assert p.step([(0.0, 1.0), (1e30, 1.0)]) is True
    assert [s for _, s in p.log] == [False, False, False, False, True]


def test_a_full_forward_after_skips_restarts_the_run():
    p = StepCachePolicy(0.5, 1)
    assert _run(p, [None, 0.1, 0.1, 0.9, 0.1]) == [False, True, False, False, True]


@pytest.mark.parametrize("threshold,cap", [(-1.0, None), (math.nan, None), (0.1, -1), (0.1, 1.5)])
def test_bad_settings(threshold, cap):
    with pytest.raises(ValueError):
        StepCachePolicy(threshold, cap)


# ------------------------------------------------------------------------------------------------ oracle
def _oracle_setup(kind):
    from diffusionkit_b200.config import tiny_flux_config, tiny_sd3_config
    from diffusionkit_b200.weights import init_params, mmdit_param_specs
    from tests.oracle_bridge import ref_config

    cfg, dtype = (tiny_flux_config(), torch.bfloat16) if kind == "flux" else (tiny_sd3_config(), torch.float16)
    p = {k: v.to(dtype).float() for k, v in init_params(mmdit_param_specs(cfg), seed=7, dtype=torch.float32).items()}
    return cfg, ref_config(cfg), p, dtype


def test_split_oracle_is_the_oracle():
    from oracle.mmdit_ref import MMDiTRef
    from tests.step_cache_ref import SplitMMDiTRef

    for kind in ("flux", "sd3"):
        cfg, rcfg, p, _ = _oracle_setup(kind)
        g = torch.Generator().manual_seed(5)
        latent = torch.randn((2, 8, 12, 16), generator=g)
        text = torch.randn((2, 16, cfg.token_level_text_embed_dim), generator=g)
        pooled = torch.randn((2, cfg.pooled_text_embed_dim), generator=g)
        t = torch.tensor([752.0])
        outs = []
        for Ref in (MMDiTRef, SplitMMDiTRef):
            ref = Ref(rcfg, p)
            ref.cache_modulation_params(pooled, t)
            outs.append(ref(latent, text, t.repeat(2)))
        assert torch.equal(outs[0], outs[1]), kind


def _loop(kind, **rule):
    from oracle import sampler_ref as sr
    from tests.step_cache_ref import SplitMMDiTRef, StepCacheRef

    cfg, rcfg, p, dtype = _oracle_setup(kind)
    steps, cfgw, shift = (6, 0.0, 1.0) if kind == "flux" else (6, 5.0, 3.0)
    sampler = sr.FluxSamplerRef(shift) if kind == "flux" else sr.ModelSamplingDiscreteFlowRef(shift)
    sig = sr.get_sigmas(sampler, steps)
    g = torch.Generator().manual_seed(3)
    reps = 2 if cfgw > 0 else 1
    cond = torch.randn((2 * reps, 16, cfg.token_level_text_embed_dim), generator=g)
    pooled = torch.randn((2 * reps, cfg.pooled_text_embed_dim), generator=g)
    x0 = torch.cat([sampler.noise_scaling(float(sig[0]), sr.get_noise(s, 8, 8), sr.get_empty_latent(8, 8))
                    for s in (11, 12)])
    model = StepCacheRef(SplitMMDiTRef(rcfg, p), **rule)
    x = sr.sample_euler(model, model.cache_modulation_params, x0, sig, cond, pooled, cfgw, dtype)
    return x, model.log


@pytest.mark.parametrize("kind", ["flux", "sd3"])
def test_oracle_replay_agrees_with_its_own_decisions(kind):
    # threshold 0 never skips: the plain loop.  A cap makes a fixed pattern; an intermediate threshold decides by rel.
    for rule in (dict(threshold=0.0), dict(threshold=math.inf, max_consecutive_skips=2), dict(threshold=0.3)):
        x_self, log_self = _loop(kind, **rule)
        x_replay, log_replay = _loop(kind, decisions=[s for _, s in log_self])
        assert torch.equal(x_self, x_replay), rule
        assert log_self == log_replay, rule
        assert log_self[0] == (None, False)
    skips = [s for _, s in _loop(kind, threshold=math.inf, max_consecutive_skips=2)[1]]
    assert skips == [False, True, True, False, True, True]
