#!/usr/bin/env python
"""CPU emulation of the device numerics contract (DESIGN.md §2) against the fp32 oracle.

TEST/ANALYSIS TOOL — not on any product path.  It restates the engine's arithmetic with torch-CPU ops:
GEMM / attention operands rounded to a 16-bit type (bf16 or fp16; optionally split into hi+lo terms), fp32
accumulation, fp32 residual stream / statistics / softmax, LayerNorm folded into the consuming GEMM exactly as
the GEMM epilogue computes it (``rstd * (r(x) W'^T - mean colsum) + b'``, one-pass variance) or, for comparison,
applied before the operand rounding (``r(LN(x)) r(W)^T``).  It answers, without a GPU:

  1. which end-to-end |dlogits_per_image| / embedding cosine each operand format can reach (north_star asks 1e-3 / 1e-4);
  2. whether the LayerNorm fold loses precision on trained-CLIP-like residual streams (``mode="outlier"`` weights);
  3. what a "centred" fold (operand = r(x - shift_r)) buys.

    python tools/precision_study.py [--images 64 --captions 32 --out precision_study.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import clip_oracle as O  # noqa: E402
from plip_b200 import synthetic as S  # noqa: E402

EPS = 1e-5


def rnd(x, fmt):
    """Operand rounding.  fmt: 'bf16' | 'fp16' | 'bf16x2' | 'fp16x2' (hi + lo split terms) | 'fp32'."""
    if fmt == "fp32":
        return x
    dt = torch.bfloat16 if fmt.startswith("bf16") else torch.float16
    hi = x.to(dt).to(torch.float32)
    if fmt.endswith("x2"):
        hi = hi + (x - hi).to(dt).to(torch.float32)
    return hi


class Cfg:
    def __init__(self, act="bf16", wgt="bf16", fold=True, centred=False, attn=None):
        self.act, self.wgt, self.fold, self.centred = act, wgt, fold, centred
        self.attn = attn or act

    def name(self):
        return f"act={self.act} wgt={self.wgt} attn={self.attn} fold={'centred' if self.centred else self.fold}"


def ln_linear(x, gamma, beta, w, b, c: Cfg, shift=None):
    """LayerNorm followed by a Linear, the way the device computes it."""
    if not c.fold:
        return rnd(O.layer_norm(x, gamma, beta), c.act) @ rnd(w, c.wgt).t() + b
    K = x.shape[-1]
    mean = x.sum(-1, keepdim=True) / K
    var = (x * x).sum(-1, keepdim=True) / K - mean * mean          # one-pass, fp32 (gemm_wgmma.cu epilogue)
    rstd = torch.rsqrt(var.clamp_min(0) + EPS)
    wf = rnd(w * gamma[None, :], c.wgt)
    colsum = wf.sum(1)
    bf = b + w @ beta
    if c.centred:
        s = shift if shift is not None else torch.zeros_like(mean)
        acc = rnd(x - s, c.act) @ wf.t()
        return rstd * (acc - (mean - s) * colsum) + bf
    acc = rnd(x, c.act) @ wf.t()
    return rstd * (acc - mean * colsum) + bf


def layer(x, sd, p, heads, mask, c: Cfg, shift):
    B, Sq, D = x.shape
    dh = D // heads
    a = f"{p}.self_attn"
    wqkv = torch.cat([sd[f"{a}.q_proj.weight"] * 0.125, sd[f"{a}.k_proj.weight"], sd[f"{a}.v_proj.weight"]], 0)
    bqkv = torch.cat([sd[f"{a}.q_proj.bias"] * 0.125, sd[f"{a}.k_proj.bias"], sd[f"{a}.v_proj.bias"]], 0)
    qkv = ln_linear(x, sd[f"{p}.layer_norm1.weight"], sd[f"{p}.layer_norm1.bias"], wqkv, bqkv, c, shift)
    qkv = rnd(qkv, c.attn)                                         # QKV activation is stored in 16 bits
    q, k, v = (t.view(B, Sq, heads, dh).transpose(1, 2) for t in qkv.split(D, dim=-1))
    s = q @ k.transpose(-1, -2)
    if mask is not None:
        s = s + mask
    mx = s.max(-1, keepdim=True).values
    e = torch.exp(s - mx)
    o = (rnd(e, c.attn) @ v) / e.sum(-1, keepdim=True)             # P rounded, row sum in fp32 (attention.cu)
    o = rnd(o.transpose(1, 2).reshape(B, Sq, D), c.act)
    x_prev_mean = x.mean(-1, keepdim=True)
    x = x + o @ rnd(sd[f"{a}.out_proj.weight"], c.wgt).t() + sd[f"{a}.out_proj.bias"]
    m = f"{p}.mlp"
    h = ln_linear(x, sd[f"{p}.layer_norm2.weight"], sd[f"{p}.layer_norm2.bias"], sd[f"{m}.fc1.weight"], sd[f"{m}.fc1.bias"],
                  c, x_prev_mean)
    h = rnd(O.quick_gelu(h), c.act)
    x_prev_mean = x.mean(-1, keepdim=True)
    x = x + h @ rnd(sd[f"{m}.fc2.weight"], c.wgt).t() + sd[f"{m}.fc2.bias"]
    return x, x_prev_mean


def towers(sd, px, ids, mask, c: Cfg):
    # vision (engine.cu vision_pass)
    B = px.shape[0]
    w = sd["vision_model.embeddings.patch_embedding.weight"]
    patches = px.reshape(B, 3, 7, 32, 7, 32).permute(0, 2, 4, 1, 3, 5).reshape(B, 49, 3072)
    pe = rnd(patches, c.act) @ rnd(w.reshape(768, -1), c.wgt).t()
    x = torch.cat([sd["vision_model.embeddings.class_embedding"].expand(B, 1, 768), pe], 1)
    x = x + sd["vision_model.embeddings.position_embedding.weight"][None]
    x = O.layer_norm(x, sd["vision_model.pre_layrnorm.weight"], sd["vision_model.pre_layrnorm.bias"])
    shift = x.mean(-1, keepdim=True)
    for i in range(12):
        x, shift = layer(x, sd, f"vision_model.encoder.layers.{i}", 12, None, c, shift)
    pooled = O.layer_norm(x[:, 0], sd["vision_model.post_layernorm.weight"], sd["vision_model.post_layernorm.bias"])
    img = rnd(pooled, c.act) @ rnd(sd["visual_projection.weight"], c.wgt).t()
    # text (engine.cu text_pass)
    x = O.text_embeddings(sd, ids)
    m = O.causal_mask(ids.shape[-1], mask)
    shift = x.mean(-1, keepdim=True)
    for i in range(12):
        x, shift = layer(x, sd, f"text_model.encoder.layers.{i}", 8, m, c, shift)
    x = O.layer_norm(x, sd["text_model.final_layer_norm.weight"], sd["text_model.final_layer_norm.bias"])
    pos = (ids == S.EOS).int().argmax(-1)
    txt = rnd(x[torch.arange(x.shape[0]), pos], c.act) @ rnd(sd["text_projection.weight"], c.wgt).t()
    return img, txt


def report(sd, ref, px, ids, mask, c: Cfg, scale):
    t0 = time.time()
    img, txt = towers(sd, px, ids, mask, c)
    ci = (1 - O.cosine(img, ref["img"])).max().item()
    ct = (1 - O.cosine(txt, ref["txt"])).max().item()
    lg = O.similarity(O.l2_normalize(img), O.l2_normalize(txt), scale)
    d = (lg - ref["logits"]).abs()
    return {"config": c.name(), "one_minus_cos_image_max": ci, "one_minus_cos_text_max": ct,
            "dlogits_max": d.max().item(), "dlogits_mean": d.mean().item(), "seconds": round(time.time() - t0, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--captions", type=int, default=32)
    ap.add_argument("--out", default="precision_study.json")
    ap.add_argument("--modes", default="rich,outlier")
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    px = S.pixel_values(args.images)
    ids, mask = S.token_ids(args.captions)
    out = {"inputs": {"images": args.images, "captions": args.captions, "pixel_seed": 1234, "ids_seed": 1235}}
    cfgs = [
        Cfg("bf16", "bf16", fold=False), Cfg("bf16", "bf16", fold=True), Cfg("bf16", "bf16", fold=True, centred=True),
        Cfg("fp16", "fp16", fold=False), Cfg("fp16", "fp16", fold=True), Cfg("fp16", "fp16", fold=True, centred=True),
        Cfg("fp16x2", "fp16", fold=True), Cfg("fp16x2", "fp16x2", fold=True), Cfg("bf16x2", "bf16x2", fold=True),
    ]
    for mode in args.modes.split(","):
        sd = S.make_state_dict(0, mode)
        scale = float(sd["logit_scale"].exp())
        ref_img, ref_txt = O.get_image_features(sd, px), O.get_text_features(sd, ids, mask)
        ref = {"img": ref_img, "txt": ref_txt,
               "logits": O.similarity(O.l2_normalize(ref_img), O.l2_normalize(ref_txt), scale)}
        hid = []
        O.vision_transformer(sd, px[:4], hidden=hid)
        rows = []
        stream = {"vision_abs_max_by_layer": [float(h.abs().max()) for h in hid],
                  "vision_row_mean_over_std_last": float((hid[-1].mean(-1).abs() / hid[-1].std(-1)).max())}
        print(mode, "residual stream:", json.dumps(stream))
        for c in cfgs:
            r = report(sd, ref, px, ids, mask, c, scale)
            r["dlogits_max_at_scale_100"] = r["dlogits_max"] * 100.0 / scale
            rows.append(r)
            print(mode, json.dumps(r), flush=True)
        out[mode] = {"logit_scale_exp": scale, "residual_stream": stream, "rows": rows}
    json.dump(out, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
