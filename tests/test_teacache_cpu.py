"""TeaCache without a GPU (-m "not gpu").

(1) The rule: the policy module (chronoedit_b200/teacache.py) and the oracle restatement (oracle/teacache_oracle.py) reproduce
    every decision and accumulator the UNMODIFIED reference class recorded (tests/golden/TEACACHE_MANIFEST.json), including
    the step counter's wrap, and the restated coefficient table equals the reference's.
(2) The mirror's state machine with its two native seams (the probe and the forward with / without blocks) stood in for by the
    oracle, as tests/test_pipeline_cpu.py does for the plain forward: separate cond / uncond states, the forced compute on a
    geometry change, the resets, and the refusals.
(3) With the same stand-ins, the unmodified reference pipeline runs the temporal-reasoning cut with TeaCache on, and its video
    equals the oracle pipeline's under the mirror's skip schedule.
"""
import json
import os

import pytest
import torch
from safetensors.torch import load_file

from chronoedit_b200 import teacache as TCP
from chronoedit_b200._lib import CEError
from oracle import cases, pipeline_cases as PC, ref_loader, teacache_oracle as TC

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MAN = json.load(open(os.path.join(GOLDEN, "TEACACHE_MANIFEST.json")))
needs_ref = pytest.mark.skipif(not ref_loader.reference_available(), reason="/root/reference only exists in the build container")


def test_coefficient_table_equals_the_reference():
    assert TCP.COEFFICIENTS == MAN["coefficients"]
    with pytest.raises(ValueError, match="Wan2.1-I2V-14B-720P"):
        TCP.TeaCacheState(50, 0.2, "Wan2.1-I2V-14B-1080P")


@needs_ref
def test_coefficient_table_equals_the_live_reference():
    from tests.golden.make_golden_teacache import reference_teacache_class

    assert TCP.COEFFICIENTS == reference_teacache_class()(1, 0.1, TCP.DEFAULT_MODEL_ID).coefficients_dict


@pytest.mark.parametrize("key", sorted(MAN["cases"]))
def test_policy_and_oracle_reproduce_the_reference(key):
    c = MAN["cases"][key]
    seq = load_file(os.path.join(GOLDEN, "teacache_tmod.safetensors"))[c["schedule"]]
    calls = list(seq) + list(seq)
    ora = TC.rule(calls, c["thresh"], c["steps"], MAN["coefficients"][c["model_id"]])
    assert [o["computed"] for o in ora] == c["computed"] and [o["acc"] for o in ora] == c["acc"]
    pol = TCP.TeaCacheState(c["steps"], c["thresh"], c["model_id"])
    prev = None
    for k, t_mod in enumerate(calls):
        rel = TC.rel_l1(t_mod, prev) if pol.needs_rel() else None
        step, computed = pol.decide(rel)
        assert (step, computed, pol.acc) == (k % c["steps"], c["computed"][k], c["acc"][k]), k
        prev = t_mod


def test_rel_from_sums_rounds_like_the_bf16_tensor_expression():
    # exact fp32 sums: |a - b| and |b| are small bf16 integers here, so only the mean's and quotient's roundings matter
    g = torch.Generator().manual_seed(0)
    for n in (6 * 256, 6 * 5120 * 2):
        b = torch.randint(1, 60, (n,), generator=g).to(torch.bfloat16)
        a = b + torch.randint(-3, 4, (n,), generator=g).to(torch.bfloat16)
        sd, sp = float((a - b).abs().float().sum()), float(b.abs().float().sum())
        f = torch.tensor(1.0 / n, dtype=torch.float32)
        num = (torch.tensor(sd, dtype=torch.float32) * f).to(torch.bfloat16)
        den = (torch.tensor(sp, dtype=torch.float32) * f).to(torch.bfloat16)
        assert TCP.rel_from_sums(sd, sp, n) == (num / den).item()


# ---------------------------------------------------------------------------------------------------------------------
# (2) the mirror's state machine with the native seams stood in for by the oracle
# ---------------------------------------------------------------------------------------------------------------------
def _mirror(dsd=None):
    import chronoedit_b200 as ce

    cfg = PC.DIT_CFG
    m = ce.ChronoEditTransformer3DModel(
        patch_size=cfg.patch_size, num_attention_heads=cfg.num_attention_heads, attention_head_dim=cfg.attention_head_dim,
        in_channels=cfg.in_channels, out_channels=cfg.out_channels, text_dim=cfg.text_dim, freq_dim=cfg.freq_dim, ffn_dim=cfg.ffn_dim,
        num_layers=cfg.num_layers, eps=cfg.eps, image_dim=cfg.image_dim, added_kv_proj_dim=cfg.added_kv_proj_dim)
    m.load_state_dict(cases.to_bf16_state(dsd if dsd is not None else PC.weights()[0]))
    m.tproj_seen = []

    def native_probe(t, prev, cur):   # stands in for ce_dit_teacache_probe (+ the pinned read of its two sums)
        cur.copy_(TC.time_modulation(dict(m.state_dict()), cfg, t).flatten())
        m.tproj_seen.append(cur.clone())
        if prev is None:
            return None
        return float((cur - prev).abs().float().sum()), float(prev.abs().float().sum())

    def native_teacache_forward(x, t, txt, img, out, txt_in, img_in, resid, record):   # ce_dit_forward_ex / ce_dit_forward_cached
        sd = dict(m.state_dict())
        if record:
            y, x0, xl = TC.forward_parts(sd, cfg, x, t, txt, img)
            resid.copy_((xl - x0).flatten())
        else:
            y, _, _ = TC.forward_parts(sd, cfg, x, t, txt, img, residual=resid.view(x.shape[0], -1, cfg.inner_dim))
        out.copy_(y)

    m._native_probe, m._native_teacache_forward = native_probe, native_teacache_forward
    return m


def _inputs(T=2, seed=0):
    g = torch.Generator().manual_seed(seed)
    cfg = PC.DIT_CFG
    x = torch.randn(1, cfg.in_channels, T, 8, 8, generator=g)
    txt = [torch.randn(1, 16, cfg.text_dim, generator=g) for _ in range(2)]
    img = torch.randn(1, 257, cfg.image_dim, generator=g)
    return x, txt, img


def test_cond_and_uncond_get_separate_states():
    m = _mirror()
    m.enable_teacache(1e9, num_inference_steps=4)   # every evaluated step would skip
    x, (cond, uncond), img = _inputs()
    for t in (900, 700, 500, 300):
        for txt in (cond, uncond):
            m(x, torch.tensor([t]), txt, img, return_dict=False)
    r = m.teacache_records
    assert [(e.slot, e.step) for e in r] == [(s, k) for k in range(4) for s in (0, 1)]
    assert [e.computed for e in r] == [True, True, False, False, False, False, True, True]
    assert r[0].rel is None and r[2].rel is not None and r[2].rel == r[3].rel   # same timesteps, same modulation


def test_geometry_change_forces_a_compute():
    m = _mirror()
    m.enable_teacache(1e9, num_inference_steps=5)
    x8, (cond, _), img = _inputs(T=8)
    x2 = x8[:, :, [0, -1]]
    for k, (t, x) in enumerate(zip((900, 800, 700, 600, 500), (x8, x8, x2, x2, x2))):
        m(x, torch.tensor([t]), cond, img)
    r = m.teacache_records
    assert [e.computed for e in r] == [True, False, True, False, True]
    assert r[2].rel is not None and r[2].acc == 0.0


@pytest.mark.parametrize("how", ["to", "load_state_dict", "load_state_dict_assign", "fuse_lora", "enable_fp8", "reset"])
def test_state_is_dropped(how):
    m = _mirror()
    m.enable_teacache(1e9, num_inference_steps=4)
    x, (cond, _), img = _inputs()
    m(x, torch.tensor([900]), cond, img)
    m(x, torch.tensor([800]), cond, img)
    if how == "to":
        m.to("cpu")
    elif how == "load_state_dict":
        m.load_state_dict(dict(m.state_dict()))
    elif how == "load_state_dict_assign":
        m.load_state_dict({k: v.clone() for k, v in m.state_dict().items()}, assign=True)
    elif how == "fuse_lora":
        w = m.blocks[0].ffn.net[2].weight
        m.fuse_lora({"blocks.0.ffn.net.2.lora_A.weight": torch.zeros(2, w.shape[1], dtype=torch.bfloat16),
                     "blocks.0.ffn.net.2.lora_B.weight": torch.zeros(w.shape[0], 2, dtype=torch.bfloat16)})
    elif how == "enable_fp8":
        m.enable_fp8()
        return   # the stand-ins read bf16 weights; that the states are gone is all there is to check
    else:
        m.reset_teacache()
    assert m._tc_states == []
    m(x, torch.tensor([700]), cond, img)
    assert m.teacache_records[-1].step == 0 and m.teacache_records[-1].computed


def test_refusals():
    m = _mirror()
    with pytest.raises(ValueError, match="supported TeaCache model id.*Wan2.1-T2V-1.3B"):
        m.enable_teacache(0.2, 50, tea_cache_model_id="nope")
    m.enable_teacache(0.2, num_inference_steps=4)
    x, (cond, _), img = _inputs()
    with pytest.raises(CEError, match="TeaCache"):
        m(x, torch.tensor([900]), cond, img, return_block0=True)
    with pytest.raises(CEError, match="TeaCache"):
        m(x, torch.tensor([900]), cond, img, capture_layers=(1,))
    m._sp_state = object()
    with pytest.raises(CEError, match="sequence parallelism"):
        m(x, torch.tensor([900]), cond, img)
    m._sp_state = None
    assert m.teacache_records == ()
    m.disable_teacache()
    assert not m.teacache_enabled


@needs_ref
def test_unmodified_pipeline_runs_the_temporal_reasoning_cut_with_teacache():
    case = PC.PIPELINE_CASES["reason_cut"]
    dsd, _ = PC.weights()
    from tests.test_pipeline_cpu import _mirror_scheduler, _mirror_vae

    tr = _mirror(dsd)
    tr.enable_teacache(1e9, num_inference_steps=case.steps)
    got = PC.run_reference_pipeline(case, torch.bfloat16, transformer=tr, vae=_mirror_vae(PC.weights()[1]),
                                    scheduler=_mirror_scheduler(case.sched_shift))
    r = tr.teacache_records
    computed = [e.computed for e in r]
    # steps 1 (cond, uncond) skip, the cut at step 2 forces a compute, step 3 is the last
    assert computed == [True, True, False, False, True, True, True, True]
    want = PC.run_oracle_pipeline(case, torch.bfloat16, transformer=TC.ScheduledTransformer(cases.to_bf16_state(dsd), PC.DIT_CFG,
                                                                                              torch.bfloat16, computed))
    assert torch.equal(got, want)
