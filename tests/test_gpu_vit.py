"""GPU: OnePeaceViT against the reference's own models_vit.py (tests/golden/vit.pt, made by oracle/make_golden_vit.py): logits
(cosine > 0.999), loss (3e-3 relative, the classification tests' bar) and every parameter gradient against its golden summary
(norm within 5 %, cosine >= 0.97 over the summary's first 256 values).  The head kernels against tests/vit_ref.py's fp64 bounds
at d = 256 and 1536, S = 17 to 1025, B = 1 to 64.  The 40-layer d = 1536 model at 384^2 against an fp32 torch restatement on
the same GPU, after a strict load of a synthetic full state dict.  autocast invariance, the criteria at C = 19167, and twenty
AdjustAdam steps with layer decay on a separable task."""
import os

import pytest
import torch
import torch.nn.functional as F

import synth
import synth_vit as sv
import vit_ref as V

pytestmark = pytest.mark.gpu
LOSS_RTOL = 3e-3


def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def _gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "vit.pt"), weights_only=False)


def _tiny(bucket, pool, **kw):
    from one_peace_b200.vision.models_vit import OnePeaceViT
    m = OnePeaceViT(bucket_size=bucket, global_pool=pool, num_classes=kw.pop("num_classes", sv.NUM_CLASSES), **sv.VIT_TINY, **kw)
    shapes = {k: tuple(p.shape) for k, p in m.named_parameters()}
    m.load_state_dict(sv.vit_state_dict(shapes, dict(m.named_buffers())), strict=True)
    return m.cuda()


@pytest.mark.parametrize("case", list(sv.VIT_CASES))
def test_vit_vs_reference(case, golden_dir):
    need_gpu()
    rec = _gold(golden_dir)["cases"][case]
    bucket, pool, crit = sv.VIT_CASES[case]
    m = _tiny(bucket, pool)
    img, soft, labels = (t.cuda() for t in sv.vit_inputs(bucket))
    m.eval()
    with torch.no_grad():
        logits = m(img)
    assert logits.dtype == torch.float32 and logits.shape == (sv.BATCH, sv.NUM_CLASSES)
    assert F.cosine_similarity(logits.flatten().cpu().double(), rec["logits"].flatten().double(), dim=0) > 0.999
    from one_peace_b200.vision.losses import LabelSmoothingCrossEntropy, SoftTargetCrossEntropy
    criterion = SoftTargetCrossEntropy() if crit == "soft" else LabelSmoothingCrossEntropy(sv.SMOOTHING)
    m.train()
    m.zero_grad(set_to_none=True)
    loss = criterion(m(img), soft if crit == "soft" else labels)
    loss.backward()
    assert abs(loss.item() - rec["loss"].item()) <= LOSS_RTOL * abs(rec["loss"].item())
    bad, n = [], 0
    for name, p in m.named_parameters():
        ref = rec["grads"][name]
        if ref["norm"] == 0:
            continue
        got = synth.grad_summary(name, p.grad.float().cpu())
        cos = F.cosine_similarity(got["head"].double(), ref["head"].double(), dim=0).item()
        ratio = got["norm"] / ref["norm"]
        n += 1
        if cos < 0.97 or abs(ratio - 1) > 0.05:
            bad.append((name, round(cos, 4), round(ratio, 4)))
    assert not bad, bad
    assert n == len(rec["grads"]) - sum(r["norm"] == 0 for r in rec["grads"].values()) and n > 40


HEAD_SHAPES = [(1, 17, 256), (3, 257, 256), (64, 577, 256), (5, 785, 256), (2, 1025, 256),
               (1, 17, 1536), (16, 257, 1536), (8, 577, 1536), (2, 785, 1536), (64, 1025, 1536)]


@pytest.mark.parametrize("B,S,d", HEAD_SHAPES)
def test_head_kernels_within_bounds(B, S, d):
    need_gpu()
    from one_peace_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(B * S + d)
    pitch = d + 4 if B * S * d < 1e8 else d            # a padded row pitch where memory allows
    big = torch.randn(B, S, pitch, generator=g, device="cuda") + torch.randn(1, 1, pitch, generator=g, device="cuda")
    x = big[:, :, :d]
    gamma = 1.0 + 0.2 * torch.randn(d, generator=g, device="cuda")
    beta = 0.1 * torch.randn(d, generator=g, device="cuda")
    dy = torch.randn(B, d, generator=g, device="cuda")
    y, m, mean, rstd = K.token_mean_ln_fwd(x, gamma, beta, 1e-5)
    r = V.head_fwd(x, gamma, beta, 1e-5)
    assert V.excess(m, r["m"], r["b_m"]) <= 1.0
    assert V.excess(mean, r["mean"], r["b_mean"]) <= 1.0
    assert V.excess(rstd, r["rstd"], r["b_rstd"]) <= 1.0
    assert V.excess(y, r["y"], r["b_y"]) <= 1.0
    del r
    dx = torch.full((B, S, pitch), float("nan"), device="cuda")[:, :, :d]
    dgamma, dbeta = K.token_mean_ln_bwd(dy, m, mean, rstd, gamma, dx)
    rb = V.head_bwd(dy, m, mean, rstd, gamma, S)
    assert V.excess(dx, rb["dx"], rb["b_dx"]) <= 1.0
    assert V.excess(dgamma, rb["dgamma"], rb["b_dgamma"]) <= 1.0
    assert V.excess(dbeta, rb["dbeta"], rb["b_dbeta"]) <= 1.0
    del rb
    assert torch.equal(dx[:, 0], torch.zeros(B, d, device="cuda"))                  # CLS rows: exact zeros
    assert torch.equal(dx[:, 1:], dx[:, 1:2].expand(B, S - 1, d))                      # one value per (sample, column)
    if pitch != d:
        assert torch.isnan(dx.as_strided((B, S, 4), (S * pitch, pitch, 1), dx.storage_offset() + d)).all()  # pad untouched
    y2, m2, mean2, rstd2 = K.token_mean_ln_fwd(x, gamma, beta, 1e-5)
    assert torch.equal(y, y2) and torch.equal(m, m2) and torch.equal(mean, mean2) and torch.equal(rstd, rstd2)
    dx2 = torch.empty(B, S, d, device="cuda")
    dgamma2, dbeta2 = K.token_mean_ln_bwd(dy, m, mean, rstd, gamma, dx2)
    assert torch.equal(dx, dx2) and torch.equal(dgamma, dgamma2) and torch.equal(dbeta, dbeta2)


def _restated_logits(P, pool, img, heads, eps=1e-5):
    """models_vit.py's forward in fp32 torch on the parameters P (a name -> tensor dict)."""
    d = P["image_adapter.pos_embed"].shape[1]
    pre = "image_adapter.embed_images."

    def ln2d(x, i):
        return F.layer_norm(x.permute(0, 2, 3, 1), (x.shape[1],), P[f"{pre}{i}.layer_norm.weight"],
                            P[f"{pre}{i}.layer_norm.bias"], eps).permute(0, 3, 1, 2)
    x = F.gelu(ln2d(F.conv2d(img, P[pre + "0.weight"], P[pre + "0.bias"], stride=4), 1))
    x = F.gelu(ln2d(F.conv2d(x, P[pre + "3.weight"], P[pre + "3.bias"], stride=2), 4))
    x = F.conv2d(x, P[pre + "6.weight"], P[pre + "6.bias"], stride=2).flatten(2).transpose(1, 2)
    B = x.shape[0]
    x = torch.cat([P["image_adapter.cls_embedding"].expand(B, -1, -1), x], 1) + P["image_adapter.pos_embed"][None]
    S = x.shape[1]
    bias = F.embedding(P["image_adapter.rp_bucket"], P["image_adapter.rel_pos_table.weight"]).permute(2, 0, 1)
    i = 0
    while f"encoder.layers.{i}.gamma_1" in P:
        L = lambda n: P[f"encoder.layers.{i}.{n}"]                       # noqa: E731
        h = F.layer_norm(x, (d,), L("self_attn_layer_norm.weight"), L("self_attn_layer_norm.bias"), eps)
        q = F.linear(h, L("self_attn.q_proj.weight"), L("self_attn.q_proj.bias")) * 64 ** -0.5
        k = F.linear(h, L("self_attn.k_proj.weight"))
        v = F.linear(h, L("self_attn.v_proj.weight"), L("self_attn.v_proj.bias"))
        q, k, v = (t.view(B, S, heads, 64).transpose(1, 2) for t in (q, k, v))
        a = torch.softmax(q @ k.transpose(-1, -2) + bias[None], dim=-1) @ v
        a = F.layer_norm(a.transpose(1, 2).reshape(B, S, d), (d,), L("self_attn.ln.weight"), L("self_attn.ln.bias"), eps)
        x = x + L("gamma_1") * F.linear(a, L("self_attn.out_proj.weight"), L("self_attn.out_proj.bias"))
        h = F.layer_norm(x, (d,), L("final_layer_norm.weight"), L("final_layer_norm.bias"), eps)
        u = F.gelu(F.linear(h, L("image_ffn.0.wi_0.weight"))) * F.linear(h, L("image_ffn.0.wi_1.weight"))
        u = F.layer_norm(u, (u.shape[-1],), L("image_ffn.2.weight"), L("image_ffn.2.bias"), eps)
        x = x + L("gamma_2") * F.linear(u, L("image_ffn.3.weight"), L("image_ffn.3.bias"))
        i += 1
    if pool:
        z = F.layer_norm(x[:, 1:].mean(1), (d,), P["fc_norm.weight"], P["fc_norm.bias"], eps)
    else:
        z = F.layer_norm(x[:, 0], (d,), P["encoder.layer_norm.weight"], P["encoder.layer_norm.bias"], eps)
    return F.linear(z, P["head.weight"], P["head.bias"])


def test_4b_model_at_384_vs_fp32_restatement():
    """one_piece_g_384 (40 layers, d = 1536, S = 577: the dense-bias attention path), B = 2: forward and one backward."""
    need_gpu()
    from one_peace_b200.vision.models_vit import one_piece_g_384
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    with torch.device("cuda"):
        m = one_piece_g_384(num_classes=1000)
    shapes = {k: tuple(p.shape) for k, p in m.named_parameters()}
    sd = sv.vit_state_dict(shapes, dict(m.named_buffers()), seed=3, device="cuda")
    sd["head.weight"] = sd["head.weight"] * 0.1
    m.load_state_dict(sd, strict=True)
    del sd
    g = torch.Generator(device="cuda").manual_seed(5)
    img = torch.randn(2, 3, 384, 384, generator=g, device="cuda")
    direction = torch.randn(2, 1000, generator=g, device="cuda")
    m.eval()
    with torch.no_grad():
        eval_logits = m(img)
    m.train()
    logits = m(img)
    (logits * direction).sum().backward()
    P = {k: v.detach().clone().requires_grad_(v.is_floating_point()) for k, v in m.state_dict().items()}
    ref = _restated_logits(P, True, img, 24)
    (ref * direction).sum().backward()
    cos = lambda a, b: F.cosine_similarity(a.flatten().double(), b.flatten().double(), dim=0).item()   # noqa: E731
    assert cos(eval_logits, ref) >= 0.999 and cos(logits, ref) >= 0.999
    names = ["head.weight", "head.bias", "fc_norm.weight", "fc_norm.bias", "image_adapter.rel_pos_table.weight"]
    names += [n for n, _ in m.named_parameters() if n.startswith(("encoder.layers.0.", "encoder.layers.39."))]
    bad = [(n, round(cos(dict(m.named_parameters())[n].grad, P[n].grad), 4)) for n in names
           if cos(dict(m.named_parameters())[n].grad, P[n].grad) <= 0.99]
    assert not bad, bad


def test_autocast_leaves_the_logits_unchanged():
    need_gpu()
    for pool in (True, False):
        m = _tiny(4, pool).eval()
        img = sv.vit_inputs(4)[0].cuda()
        with torch.no_grad():
            plain = m(img)
            with torch.autocast("cuda"):                  # engine_finetune.evaluate uses torch.cuda.amp.autocast()
                auto = m(img)
        assert auto.dtype == torch.float32 and torch.equal(plain, auto)


@pytest.mark.parametrize("kind", ["soft", "smooth"])
def test_criteria_at_21k_classes(kind):
    need_gpu()
    from one_peace_b200.vision.losses import LabelSmoothingCrossEntropy, SoftTargetCrossEntropy
    C, B = 19167, 8
    g = torch.Generator(device="cuda").manual_seed(9)
    store = torch.randn(B, C + 1, generator=g, device="cuda") * 3                 # logits at a row pitch of C + 1
    logits = store[:, :C].requires_grad_(False).clone().requires_grad_(True)
    soft = torch.softmax(torch.randn(B, C, generator=g, device="cuda"), 1)
    labels = torch.randint(0, C, (B,), generator=g, device="cuda")
    x64 = logits.detach().double().requires_grad_(True)
    if kind == "soft":
        loss = SoftTargetCrossEntropy()(logits, soft)
        want = sv.soft_target_ce(x64, soft.double())
    else:
        loss = LabelSmoothingCrossEntropy(0.1)(logits, labels)
        want = sv.label_smoothing_ce(x64, labels, 0.1)
    loss.backward()
    want.backward()
    assert abs(loss.item() - want.item()) <= 1e-5 * abs(want.item())
    err = (logits.grad.double() - x64.grad).abs().max().item()
    assert err <= 1e-5 * x64.grad.abs().max().item()


def test_adjust_adam_with_layer_decay_drives_the_loss_down():
    """Twenty steps on a separable task (the class is the sign of a constant offset on the red channel), with main_ft.py's
    layer-decay groups (utils/lr_decay.param_groups_lrd, restated) at decay 0.85."""
    need_gpu()
    from types import SimpleNamespace
    from one_peace_b200.optim.adam import AdjustAdam
    from one_peace_b200.vision.losses import SoftTargetCrossEntropy
    m = _tiny(4, True, num_classes=2, drop_path_rate=0.1)
    m.train()
    g = torch.Generator().manual_seed(0)
    y = torch.arange(16) % 2
    img = torch.randn(16, 3, 64, 64, generator=g)
    img[:, 0] += torch.where(y == 1, 1.0, -1.0)[:, None, None]
    img, target = img.cuda(), F.one_hot(y, 2).float().cuda()
    n_layers = len(m.encoder.layers) + 1
    groups = {}
    for n, p in m.named_parameters():
        lid = 0 if n.startswith("image_adapter") else (int(n.split(".")[2]) + 1 if n.startswith("encoder.layers") else n_layers)
        nd = p.ndim == 1 or n in m.no_weight_decay()
        grp = groups.setdefault((lid, nd), dict(params=[], lr_scale=0.85 ** (n_layers - lid), weight_decay=0.0 if nd else 0.05))
        grp["params"].append(p)
    opt = AdjustAdam(SimpleNamespace(lr=[5e-4], adam_betas=(0.9, 0.999), adam_eps=1e-8, weight_decay=0.05), list(groups.values()))
    opt.set_lr(5e-4)
    crit = SoftTargetCrossEntropy()
    losses = []
    for _ in range(20):
        m.zero_grad(set_to_none=True)
        loss = crit(m(img), target)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < 0.5 * losses[0], losses
