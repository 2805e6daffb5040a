"""GPU bring-up: per-kernel and whole-model parity vs torch / the oracle, each section in its own
subprocess under a timeout (a trap in one section cannot take the others down)."""
import json
import subprocess
import sys
import time

import torch

SECTIONS = ["ln", "im2col", "attn_vision", "attn_text", "attn_text_mask", "similarity", "vision", "text", "host", "perf"]


def _lib():
    from plip_b200._lib import lib, check
    return lib(), check


def sec_ln():
    L, check = _lib()
    dev = "cuda"
    for D in (768, 512):
        x = torch.randn(1000, D, device=dev) * 3 + 0.5
        g = torch.randn(D, device=dev)
        b = torch.randn(D, device=dev)
        of = torch.empty_like(x)
        ob = torch.empty(1000, D, device=dev, dtype=torch.bfloat16)
        check(L.plip_dbg_layernorm(x.data_ptr(), 1000, D, D, g.data_ptr(), b.data_ptr(), of.data_ptr(), ob.data_ptr(),
                                   torch.cuda.current_stream().cuda_stream), "ln")
        ref = torch.nn.functional.layer_norm(x, (D,), g, b, 1e-5)
        print(json.dumps({"ln_D": D, "f32_err": (of - ref).abs().max().item(),
                          "bf16_err": (ob.float() - ref).abs().max().item()}))


def sec_im2col():
    L, check = _lib()
    from oracle import clip_oracle as O
    dev = "cuda"
    n = 5
    px = torch.randn(n, 3, 224, 224, device=dev)
    ref = px.reshape(n, 3, 7, 32, 7, 32).permute(0, 2, 4, 1, 3, 5).reshape(n * 49, 3072)
    st = torch.cuda.current_stream().cuda_stream
    out = torch.empty(n * 49, 3072, device=dev, dtype=torch.bfloat16)
    check(L.plip_dbg_im2col(px.data_ptr(), 0, n, out.data_ptr(), st), "im2col f32")
    e0 = (out.float() - ref.to(torch.bfloat16).float()).abs().max().item()
    pb = px.to(torch.bfloat16)
    check(L.plip_dbg_im2col(pb.data_ptr(), 1, n, out.data_ptr(), st), "im2col bf16")
    e1 = (out.float() - ref.to(torch.bfloat16).float()).abs().max().item()
    u8 = torch.randint(0, 256, (n, 224, 224, 3), dtype=torch.uint8)
    pref = O.preprocess_u8(u8).to(dev)
    ref8 = pref.reshape(n, 3, 7, 32, 7, 32).permute(0, 2, 4, 1, 3, 5).reshape(n * 49, 3072)
    u8d = u8.to(dev)
    check(L.plip_dbg_im2col(u8d.data_ptr(), 2, n, out.data_ptr(), st), "im2col u8")
    e2 = (out.float() - ref8).abs().max().item()
    print(json.dumps({"im2col_f32": e0, "im2col_bf16": e1, "im2col_u8_vs_f32ref": e2}))


def _attn(n_seq, S, heads, causal, use_mask):
    L, check = _lib()
    dev = "cuda"
    D = heads * 64
    g = torch.Generator().manual_seed(3)
    qkv = (torch.randn(n_seq * S, 3 * D, generator=g)).to(dev).to(torch.bfloat16)
    out = torch.zeros(n_seq * S, D, device=dev, dtype=torch.bfloat16)
    mask = None
    if use_mask:
        lens = torch.randint(3, S + 1, (n_seq,), generator=g)
        mask = (torch.arange(S)[None] < lens[:, None]).to(torch.int32).to(dev).contiguous()
    check(L.plip_dbg_attention(qkv.data_ptr(), n_seq, S, heads, int(causal), mask.data_ptr() if mask is not None else None,
                               out.data_ptr(), torch.cuda.current_stream().cuda_stream), "attention")
    torch.cuda.synchronize()
    q, k, v = qkv.float().view(n_seq, S, 3, heads, 64).permute(2, 0, 3, 1, 4)
    att = q @ k.transpose(-1, -2)  # scale folded into q by the packer; raw test data here -> no scale
    neg = float("-inf")
    if causal:
        att = att + torch.full((S, S), neg, device=dev).triu(1)
    if mask is not None:
        att = att.masked_fill((mask == 0)[:, None, None, :], neg)
    p = torch.softmax(att, -1)
    ref = (p @ v).permute(0, 2, 1, 3).reshape(n_seq * S, D)
    err = (out.float() - ref).abs()
    if mask is not None:  # rows whose query is itself padding are don't-care only if fully masked; compare all finite
        pass
    print(json.dumps({"attn": [n_seq, S, heads, causal, use_mask], "max_err": err.max().item(),
                      "mean_err": err.mean().item(), "ref_max": ref.abs().max().item(),
                      "nan": bool(torch.isnan(out.float()).any())}))


def sec_attn_vision():
    _attn(7, 50, 12, False, False)
    _attn(64, 50, 12, False, False)


def sec_attn_text():
    _attn(5, 77, 8, True, False)
    _attn(33, 77, 8, True, False)
    _attn(6, 20, 8, True, False)


def sec_attn_text_mask():
    _attn(9, 77, 8, True, True)


def sec_similarity():
    L, check = _lib()
    dev = "cuda"
    a = torch.randn(300, 512, device=dev)
    b = torch.randn(70, 512, device=dev)
    out = torch.empty(300, 72, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    import ctypes as C
    check(L.plip_similarity(a.data_ptr(), 300, b.data_ptr(), 70, C.c_float(14.3), 1, 1, out.data_ptr(), 72, st), "sim")
    an = a.double() / a.double().norm(dim=-1, keepdim=True)
    bn = b.double() / b.double().norm(dim=-1, keepdim=True)
    ref = (14.3 * an @ bn.t()).float()
    e = (out[:, :70] - ref).abs().max().item()
    idx = torch.empty(300, 5, device=dev, dtype=torch.int32)
    val = torch.empty(300, 5, device=dev)
    check(L.plip_similarity_topk(a.data_ptr(), 300, b.data_ptr(), 70, C.c_float(14.3), 1, 1, 5, idx.data_ptr(),
                                 val.data_ptr(), st), "topk")
    rv, ri = ref.topk(5, dim=-1)
    print(json.dumps({"sim_err": e, "topk_idx_match": bool((ri.int() == idx).all()), "topk_val_err": (rv - val).abs().max().item()}))


def _engine(max_mb=64):
    from oracle import weights
    from plip_b200.engine import Engine
    sd = weights.make_state_dict(0)
    return sd, Engine(sd, max_micro_batch=max_mb)


def sec_vision():
    from oracle import clip_oracle as O, synth
    sd, eng = _engine()
    n = 6
    px = synth.pixel_values(n)
    hid = []
    pooled = O.vision_transformer(sd, px, hidden=hid)
    ref = O.get_image_features(sd, px)
    for nl in (0, 1, 2, 6, 12):
        h = eng.hidden_states("vision", px.cuda(), nl).cpu()
        d = (h - hid[nl]).abs()
        print(json.dumps({"vision_hidden_layers": nl, "max_err": d.max().item(), "mean_err": d.mean().item(),
                          "ref_absmax": hid[nl].abs().max().item()}))
    out = eng.encode_images(px.cuda()).cpu()
    print(json.dumps({"vision_embed_1-cos_max": (1 - O.cosine(out, ref)).max().item(),
                      "abs_err": (out - ref).abs().max().item(), "ref_absmax": ref.abs().max().item()}))
    u8 = torch.from_numpy(synth.tiles_u8(n))
    ref8 = O.get_image_features(sd, O.preprocess_u8(u8))
    out8 = eng.encode_images(u8.cuda()).cpu()
    print(json.dumps({"vision_u8_embed_1-cos_max": (1 - O.cosine(out8, ref8)).max().item()}))


def sec_text():
    from oracle import clip_oracle as O, synth
    sd, eng = _engine()
    n = 6
    ids, mask = synth.token_ids(n)
    hid = []
    O.text_transformer(sd, ids, mask, hidden=hid)
    ref = O.get_text_features(sd, ids, mask)
    for nl in (0, 1, 12):
        h = eng.hidden_states("text", ids.cuda(), nl, attention_mask=mask.cuda()).cpu()
        # rows after the first eos are don't-care under the padding mask? No: HF computes them too; compare all
        d = (h - hid[nl]).abs()
        print(json.dumps({"text_hidden_layers": nl, "max_err": d.max().item(), "mean_err": d.mean().item(),
                          "ref_absmax": hid[nl].abs().max().item()}))
    out = eng.encode_text(ids.cuda(), mask.cuda()).cpu()
    out_nomask = eng.encode_text(ids.cuda()).cpu()
    print(json.dumps({"text_embed_1-cos_max": (1 - O.cosine(out, ref)).max().item(),
                      "nomask_vs_mask": (out - out_nomask).abs().max().item(),
                      "abs_err": (out - ref).abs().max().item(), "ref_absmax": ref.abs().max().item()}))
    full = O.clip_forward(sd, ids, synth.pixel_values(n), mask)
    img = eng.encode_images(synth.pixel_values(n).cuda())
    txt = eng.encode_text(ids.cuda(), mask.cuda())
    lg = eng.similarity(img, txt).cpu()
    print(json.dumps({"e2e_logits_err": (lg - full["logits_per_image"]).abs().max().item(),
                      "logit_absmax": full["logits_per_image"].abs().max().item()}))


def sec_host():
    from oracle import synth
    sd, eng = _engine(max_mb=16)
    u8 = torch.from_numpy(synth.tiles_u8(50))
    a = eng.encode_images(u8.cuda()).cpu()
    b = eng.encode_images_host(u8.numpy())
    c = eng.encode_images_host(u8.pin_memory())
    ids, mask = synth.token_ids(40)
    t0 = eng.encode_text(ids.cuda(), mask.cuda()).cpu()
    t1 = eng.encode_text_host(ids, mask)
    print(json.dumps({"host_vs_dev_pageable": (a - b).abs().max().item(), "host_vs_dev_pinned": (a - c).abs().max().item(),
                      "text_host_vs_dev": (t0 - t1).abs().max().item()}))  # host path processes only the longest-caption prefix


def sec_perf():
    from oracle import synth
    sd, eng = _engine(max_mb=1024)
    for mb, fmt in ((1024, "bf16"), (1024, "u8"), (256, "bf16")):
        eng.close()
        from plip_b200.engine import Engine
        eng = Engine(sd, max_micro_batch=mb)
        n = 1024
        if fmt == "bf16":
            px = torch.randn(n, 3, 224, 224, device="cuda", dtype=torch.bfloat16)
        else:
            px = torch.randint(0, 256, (n, 224, 224, 3), device="cuda", dtype=torch.uint8)
        for _ in range(3):
            eng.encode_images(px)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            eng.encode_images(px)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 5
        print(json.dumps({"perf_vision": fmt, "micro_batch": mb, "ms_per_1024": ms, "img_per_s": n / ms * 1e3,
                          "tflops": 1024 * 8.81762e9 / ms / 1e9}))
    ids, mask = synth.token_ids(1024, full_length=True)
    ids = ids.cuda()
    for _ in range(3):
        eng.encode_text(ids)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        eng.encode_text(ids)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 5
    print(json.dumps({"perf_text": 1024, "ms": ms, "cap_per_s": 1024 / ms * 1e3, "tflops": 1024 * 5.95954e9 / ms / 1e9}))


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--section":
        globals()["sec_" + sys.argv[2]]()
        sys.exit(0)
    todo = sys.argv[1:] or SECTIONS
    for s in todo:
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, __file__, "--section", s], capture_output=True, text=True, timeout=300)
            print(f"== {s} rc={r.returncode} {time.time()-t0:.1f}s")
            print(r.stdout.strip())
            if r.returncode != 0:
                print("\n".join(r.stderr.strip().splitlines()[-12:]))
        except subprocess.TimeoutExpired:
            print(f"== {s} TIMEOUT")
        sys.stdout.flush()
