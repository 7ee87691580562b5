#!/usr/bin/env python
"""Generate the golden fixtures by running the UNMODIFIED reference in this (build) container.

    python tests/golden/make_golden.py            # writes tests/golden/*.safetensors + MANIFEST.json

Sources of truth executed here (never copied into the repo):
  * /root/reference/chronoedit_diffusers/transformer_chronoedit.py  (ChronoEditTransformer3DModel), with the
    un-vendored diffusers symbols supplied by oracle/diffusers_shim
  * /root/reference/chronoedit/_src/tokenizers/wan2pt1.py  (WanVAE_)
  * /root/reference/chronoedit_diffsynth/wan_video_dit_chronoedit.py (independent in-tree DiT modules; used
    only to corroborate the restated diffusers semantics, result recorded in MANIFEST.json)

For every case of oracle/cases.py the reference is run in fp32 and in the bf16 configuration the CLI uses
(run_inference_diffusers.py:341-353: bf16 weights, `_keep_in_fp32_modules` in fp32); the oracle restatement
must agree (fp32 <= 1e-5, bf16 bit-exact) or generation aborts.  /root/reference does not exist on the GPU
box, so the tests there read only the files written here.
"""
from __future__ import annotations

import json
import os
import sys
import time

import torch
from safetensors.torch import save_file

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import cases, dit_oracle, ref_loader, vae_oracle  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def build_reference_dit(ref, cfg: dit_oracle.DiTConfig):
    return ref.ChronoEditTransformer3DModel(
        patch_size=cfg.patch_size, num_attention_heads=cfg.num_attention_heads,
        attention_head_dim=cfg.attention_head_dim, in_channels=cfg.in_channels, out_channels=cfg.out_channels,
        text_dim=cfg.text_dim, freq_dim=cfg.freq_dim, ffn_dim=cfg.ffn_dim, num_layers=cfg.num_layers,
        cross_attn_norm=cfg.cross_attn_norm, qk_norm=cfg.qk_norm, eps=cfg.eps, image_dim=cfg.image_dim,
        added_kv_proj_dim=cfg.added_kv_proj_dim, rope_max_seq_len=cfg.rope_max_seq_len,
        rope_temporal_skip_len=cfg.rope_temporal_skip_len).eval()


def diffsynth_crosscheck(case: cases.DiTCase, sd, y_ref: torch.Tensor) -> float:
    """Run the same weights through DiffSynth's independently written modules (glued like the live
    model_fn_wan_video, but with the skip-PE temporal positions) and return max |diff| vs the reference."""
    ds = ref_loader.load_reference_diffsynth_dit()
    cfg = case.cfg
    D = cfg.inner_dim
    x, t, text, img = cases.dit_inputs(case)
    blocks = []
    for i in range(cfg.num_layers):
        b = ds.DiTBlock(True, D, cfg.num_attention_heads, cfg.ffn_dim, cfg.eps).eval()
        p = f"blocks.{i}."
        m = {
            "self_attn.q": "attn1.to_q", "self_attn.k": "attn1.to_k", "self_attn.v": "attn1.to_v",
            "self_attn.o": "attn1.to_out.0", "cross_attn.q": "attn2.to_q", "cross_attn.k": "attn2.to_k",
            "cross_attn.v": "attn2.to_v", "cross_attn.o": "attn2.to_out.0", "cross_attn.k_img": "attn2.add_k_proj",
            "cross_attn.v_img": "attn2.add_v_proj", "ffn.0": "ffn.net.0.proj", "ffn.2": "ffn.net.2",
        }
        bsd = {}
        for a, r in m.items():
            bsd[a + ".weight"] = sd[p + r + ".weight"]
            bsd[a + ".bias"] = sd[p + r + ".bias"]
        bsd["self_attn.norm_q.weight"] = sd[p + "attn1.norm_q.weight"]
        bsd["self_attn.norm_k.weight"] = sd[p + "attn1.norm_k.weight"]
        bsd["cross_attn.norm_q.weight"] = sd[p + "attn2.norm_q.weight"]
        bsd["cross_attn.norm_k.weight"] = sd[p + "attn2.norm_k.weight"]
        bsd["cross_attn.norm_k_img.weight"] = sd[p + "attn2.norm_added_k.weight"]
        bsd["norm3.weight"] = sd[p + "norm2.weight"]   # DiffSynth names the affine cross-attn norm "norm3"
        bsd["norm3.bias"] = sd[p + "norm2.bias"]
        bsd["modulation"] = sd[p + "scale_shift_table"]
        b.load_state_dict(bsd)
        blocks.append(b)
    with torch.no_grad():
        # embedders from the oracle pieces (they are checked separately against the reference run)
        temb, tproj, text_e, img_e = dit_oracle.condition_embedder(sd, cfg, t, text, img)
        ctx = torch.cat([img_e, text_e], dim=1)
        h = torch.nn.functional.conv3d(x, sd["patch_embedding.weight"], sd["patch_embedding.bias"],
                                       stride=cfg.patch_size).flatten(2).transpose(1, 2)
        f_t, f_h, f_w = ds.precompute_freqs_cis_3d(cfg.attention_head_dim)
        pf, ph_, pw_ = case.frames, case.height // 2, case.width // 2
        ft = f_t[: cfg.rope_temporal_skip_len][[0, -1]] if pf == 2 else f_t[:pf]
        freqs = torch.cat([ft.view(pf, 1, 1, -1).expand(pf, ph_, pw_, -1),
                           f_h[:ph_].view(1, ph_, 1, -1).expand(pf, ph_, pw_, -1),
                           f_w[:pw_].view(1, 1, pw_, -1).expand(pf, ph_, pw_, -1)], dim=-1).reshape(pf * ph_ * pw_, 1, -1)
        t_mod = tproj.unflatten(1, (6, D))
        for b in blocks:
            h = b(h, ctx, t_mod, freqs)
        head = ds.Head(D, cfg.out_channels, cfg.patch_size, cfg.eps).eval()
        head.load_state_dict({"head.weight": sd["proj_out.weight"], "head.bias": sd["proj_out.bias"],
                              "modulation": sd["scale_shift_table"]})
        o = head(h, temb)
        B = x.shape[0]
        o = o.reshape(B, pf, ph_, pw_, 1, 2, 2, -1).permute(0, 7, 1, 4, 2, 5, 3, 6).flatten(6, 7).flatten(4, 5).flatten(2, 3)
    return float((o - y_ref).abs().max())


def main():
    assert ref_loader.reference_available(), "run this in the build container (needs /root/reference)"
    torch.manual_seed(0)
    torch.set_num_threads(os.cpu_count() or 1)
    manifest = {"torch": torch.__version__, "generated_by": "tests/golden/make_golden.py", "cases": {}}
    ref_dit = ref_loader.load_reference_dit()
    ref_vae = ref_loader.load_reference_vae()

    for name, case in cases.DIT_CASES.items():
        t0 = time.time()
        sd = cases.dit_weights(case)
        x, t, text, img = cases.dit_inputs(case)
        m = build_reference_dit(ref_dit, case.cfg)
        assert set(m.state_dict().keys()) == set(sd.keys())
        m.load_state_dict(sd)
        with torch.no_grad():
            y32 = m(x, t, text, img, return_dict=False)[0]
            o32, inter = dit_oracle.dit_forward(sd, case.cfg, x, t, text, img, return_intermediates=True)
        d32 = float((y32 - o32).abs().max())
        assert d32 <= 1e-5, (name, d32)
        sdb = cases.to_bf16_state(sd)
        m.to(torch.bfloat16)
        m.load_state_dict(sdb, assign=True)
        xb, tb, textb, imgb = x.bfloat16(), t, text.bfloat16(), img.bfloat16()
        with torch.no_grad():
            y16 = m(xb, tb, textb, imgb, return_dict=False)[0]
            o16, inter16 = dit_oracle.dit_forward(sdb, case.cfg, xb, tb, textb, imgb, return_intermediates=True)
        assert torch.equal(y16, o16), (name, float((y16.float() - o16.float()).abs().max()))
        ds = diffsynth_crosscheck(case, sd, y32)
        assert ds <= 1e-4, (name, ds)
        tensors = {"out_fp32": y32.contiguous(), "out_bf16": y16.contiguous(),
                   "timestep_proj_fp32": inter["timestep_proj"].contiguous()}
        if inter["block0"].shape[1] <= 512:  # per-layer checkpoints only for the small cases (fixture size)
            tensors.update({
                "block0_fp32": inter["block0"].contiguous(), "block0_bf16": inter16["block0"].contiguous(),
            })
        save_file(tensors, os.path.join(OUT, f"dit_{name}.safetensors"))
        manifest["cases"][f"dit_{name}"] = {
            "oracle_vs_reference_fp32_maxabs": d32, "oracle_vs_reference_bf16_equal": True,
            "diffsynth_vs_reference_fp32_maxabs": ds,
            "bf16_vs_fp32_maxabs": float((y16.float() - y32).abs().max()),
            "bf16_vs_fp32_meanabs": float((y16.float() - y32).abs().mean()),
            "out_meanabs": float(y32.abs().mean()),
            "weights_checksum": cases.checksum(torch.cat([v.flatten()[:4096].float() for v in sd.values()])),
            "inputs_checksum": cases.checksum(torch.cat([x.flatten(), text.flatten()[:65536], img.flatten()[:65536]])),
            "seconds": round(time.time() - t0, 2),
        }
        print(name, manifest["cases"][f"dit_{name}"], flush=True)

    for name, case in cases.VAE_CASES.items():
        t0 = time.time()
        cfg = case.cfg
        sd = cases.vae_weights(case)
        video, z = cases.vae_inputs(case)
        m = ref_vae.WanVAE_(dim=cfg.dim, z_dim=cfg.z_dim, dim_mult=list(cfg.dim_mult), num_res_blocks=cfg.num_res_blocks,
                            attn_scales=[], temperal_downsample=list(cfg.temperal_downsample), dropout=0.0).eval()
        assert set(m.state_dict().keys()) == set(sd.keys())
        m.load_state_dict(sd)
        with torch.no_grad():
            mu32 = m.encode(video, [0.0, 1.0])
            dec32 = m.decode(z, [0.0, 1.0])
            omu = vae_oracle.vae_encode(sd, cfg, video)
            odec = vae_oracle.vae_decode(sd, cfg, z, clamp=False)
        e1, e2 = float((mu32 - omu).abs().max()), float((dec32 - odec).abs().max())
        assert e1 <= 1e-5 and e2 <= 1e-5, (name, e1, e2)
        mb = m.to(torch.bfloat16)
        sdb = {k: v.to(torch.bfloat16) for k, v in sd.items()}
        with torch.no_grad():
            mu16 = mb.encode(video.bfloat16(), [0.0, 1.0])
            dec16 = mb.decode(z.bfloat16(), [0.0, 1.0])
            omu16 = vae_oracle.vae_encode(sdb, cfg, video.bfloat16())
            odec16 = vae_oracle.vae_decode(sdb, cfg, z.bfloat16(), clamp=False)
        assert torch.equal(mu16, omu16) and torch.equal(dec16, odec16), name
        save_file({"mu_fp32": mu32.contiguous(), "dec_fp32": dec32.contiguous(),
                   "mu_bf16": mu16.contiguous(), "dec_bf16": dec16.contiguous()},
                  os.path.join(OUT, f"vae_{name}.safetensors"))
        manifest["cases"][f"vae_{name}"] = {
            "oracle_vs_reference_fp32_maxabs": max(e1, e2), "oracle_vs_reference_bf16_equal": True,
            "enc_bf16_vs_fp32_maxabs": float((mu16.float() - mu32).abs().max()),
            "enc_bf16_vs_fp32_meanabs": float((mu16.float() - mu32).abs().mean()),
            "dec_bf16_vs_fp32_maxabs": float((dec16.float() - dec32).abs().max()),
            "dec_bf16_vs_fp32_meanabs": float((dec16.float() - dec32).abs().mean()),
            "mu_meanabs": float(mu32.abs().mean()), "dec_meanabs": float(dec32.abs().mean()),
            "weights_checksum": cases.checksum(torch.cat([v.flatten()[:4096].float() for v in sd.values()])),
            "inputs_checksum": cases.checksum(torch.cat([video.flatten(), z.flatten()])),
            "seconds": round(time.time() - t0, 2),
        }
        print(name, manifest["cases"][f"vae_{name}"], flush=True)

    with open(os.path.join(OUT, "MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1, sort_keys=True)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
