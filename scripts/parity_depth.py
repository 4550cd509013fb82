"""Full-depth parity study (BASELINE.json configs[1] and [2]) with an error-budget control.

For the 40-layer 4B-width encoder (4 distinct seeded layers cycled) on 8 images + 8 ragged texts (+ 8 x 10 s audio with
--audio) this prints one JSON line with, per network ("conditioned": LayerScale in (1e-3, 3e-3), the regime of a trained
model whose LayerScale starts at 1e-6; "hard": LayerScale U(0.5, 1.5), residual stream dominated by random branches):

  * cosine / loss error of the sm_90a path vs the fp32 CPU oracle, with bf16 and with fp32 parameters;
  * the SAME numbers for `oracle/restated.py` run on the GPU in bf16 eager (what the reference itself does with
    `dtype=bf16`: bf16 weights, bf16 activations, bf16 residual stream, ATen / cuBLAS) — the error budget a bf16
    implementation of the reference has against its own fp32 arithmetic.

Test infrastructure (imports oracle/); tests/test_gpu_full_depth.py asserts the gates on the same construction."""
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import restated as R  # noqa: E402
import synth  # noqa: E402

D, FFN, H, L, VOCAB, B = 1536, 6144, 24, 40, 4096, 8
NETS = {"conditioned": (0.001, 0.003), "hard": (0.5, 1.5)}


def build_sd(gamma_range, layers=L, distinct=4, seed=2, modalities=("text", "image", "audio")):
    sd = synth.make_state_dict(embed_dim=D, ffn=FFN, layers=distinct, heads=H, seed=seed, vocab=VOCAB, modalities=modalities,
                               gamma_range=gamma_range)
    for i in range(distinct, layers):
        for k in [k for k in sd if f"fusion_model.layers.{i % distinct}." in k]:
            sd[k.replace(f"fusion_model.layers.{i % distinct}.", f"fusion_model.layers.{i}.")] = sd[k]
    return sd


def inputs(seed=11, n_text=B, audio=False):
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(4, VOCAB, (n_text, 71), generator=g)
    for i in range(n_text):
        tok[i, 71 - 7 * (i % 8):] = 1                            # ragged: 71, 64, ... tokens, rest padding
    img = torch.randn(B, 3, 224, 224, generator=g)
    aud = apm = None
    if audio:
        N = 160000
        aud = F.layer_norm(torch.randn(B, N, generator=g), (N,))
        T = R.audio_frames(N, R.OracleConfig().feature_encoder_spec)
        apm = torch.zeros(B, T + 1, dtype=torch.bool)
        for b, keep in ((2, 0.6), (5, 0.35)):
            aud[b, int(N * keep):] = 0.0
            apm[b, 1 + int(T * keep):] = True
    return tok, img, aud, apm


def oracle_embeddings(sd, tok, img, aud, apm, device="cpu", dtype=torch.float32):
    cfg = R.OracleConfig(embed_dim=D, ffn_embed_dim=FFN, layers=L, attention_heads=H)
    cast = lambda v: v.to(device=device, dtype=dtype) if v.is_floating_point() else v.to(device)
    sdd = {k: cast(v) for k, v in sd.items()}
    out = {}
    with torch.no_grad():
        out["text"] = R.extract_features(sdd, cfg, "text", src_tokens=tok.to(device))
        out["image"] = R.extract_features(sdd, cfg, "image", src_images=cast(img))
        if aud is not None:
            out["audio"] = R.extract_features(sdd, cfg, "audio", src_audios=cast(aud), audio_padding_masks=apm.to(device))
    return {k: v.float().cpu() for k, v in out.items()}


def losses(emb, scale):
    out = {"itc": R.itc_loss(emb["image"], emb["text"], emb["image"], emb["text"], scale, 0, 0.0)[0].item()}
    if "audio" in emb:
        out["atc"] = R.itc_loss(emb["audio"], emb["text"], emb["audio"], emb["text"], scale, 0, 0.0)[0].item()
    return out


def compare(got, want, scale):
    res = {"min_cos": {m: round(F.cosine_similarity(got[m], want[m]).min().item(), 6) for m in want}}
    lg, lw = losses(got, scale), losses(want, scale)
    res["loss_rel"] = {k: float(f"{abs(lg[k] - lw[k]) / abs(lw[k]):.3e}") for k in lw}
    ws = want["image"] @ want["text"].t()
    gs = got["image"] @ got["text"].t()
    res["i2t_argmax_equal_rows"] = int((ws.argmax(1) == gs.argmax(1)).sum())
    top2 = ws.topk(2, dim=1).values
    res["i2t_min_margin"] = round((top2[:, 0] - top2[:, 1]).min().item(), 5)
    return res


def main():
    audio = "--audio" in sys.argv
    from one_peace_b200.one_peace.hub_interface import from_pretrained
    torch.set_num_threads(min(os.cpu_count() or 1, 16))
    tok, img, aud, apm = inputs(audio=audio)
    line = {"config": f"4B width, {L} layers (4 distinct cycled), {B} images + {B} ragged texts" + (" + 8 x 10 s audio" if audio else "")}
    for name, gr in NETS.items():
        sd = build_sd(gr)
        scale = R.logit_scale_exp(sd["logit_scale"])
        want = oracle_embeddings(sd, tok, img, aud, apm)
        res = {}
        for dtype in ("bfloat16", "float32"):
            hub = from_pretrained(state_dict=sd, head_type="val", layers=L, embed_dim=D, ffn_embed_dim=FFN, attention_heads=H,
                                  patch_image_size=224, device="cuda", dtype=dtype, vocab_size=VOCAB)
            got = {"text": hub.extract_text_features(tok.cuda()).float().cpu(),
                   "image": hub.extract_image_features(img.cuda()).float().cpu()}
            if audio:
                got["audio"] = hub.extract_audio_features(aud.cuda(), apm.cuda()).float().cpu()
            res[f"repo_{dtype}_params"] = compare(got, want, scale)
            del hub
            torch.cuda.empty_cache()
        res["eager_bf16_reference_on_gpu"] = compare(oracle_embeddings(sd, tok, img, aud, apm, "cuda", torch.bfloat16), want, scale)
        torch.backends.cuda.matmul.allow_tf32 = False
        res["eager_fp32_reference_on_gpu"] = compare(oracle_embeddings(sd, tok, img, aud, apm, "cuda", torch.float32), want, scale)
        sdq = {k: (v.to(torch.bfloat16).float() if v.is_floating_point() else v) for k, v in sd.items()}
        res["oracle_fp32_with_bf16_rounded_weights"] = compare(oracle_embeddings(sdq, tok, img, aud, apm), want, scale)
        line[name] = res
    print(json.dumps(line))


if __name__ == "__main__":
    main()
