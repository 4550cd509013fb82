"""GPU: the attention-pooling forward / backward and the classification-loss kernels (csrc/classify.cu) element by element
within the fp64 references and bounds of tests/test_classify_host_logic.py; bit-identical repeats, exact zeros on padded dkv
rows, NaN in padded rows and pad columns reaching nothing, and no write outside the logical outputs."""
import math

import pytest
import torch

from test_classify_host_logic import HARD, HINGE, MULTI, SOFT, excess, loss_ref, pool_bwd_ref, pool_fwd_ref

pytestmark = pytest.mark.gpu


def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def _inputs(B, T, d, pad, q_scale, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    H = d // 64
    kv = torch.randn(B * T, 2 * d, device="cuda", generator=g).bfloat16()
    if q_scale == "init":
        q = (0.02 * torch.randn(H, 64, device="cuda", generator=g)).clamp(-0.02, 0.02)
    else:
        # scores span about +-30: |q . k| ~ |q| * 8 for unit-variance k
        q = torch.randn(H, 64, device="cuda", generator=g) * (30.0 / 8.0 / 8.0) * 2
    kp = None
    if pad == "ragged":
        kp = torch.zeros(B, T, dtype=torch.uint8, device="cuda")
        for b in range(B):
            kp[b, T - (b * 7) % T:] = 1 if b % T else 0
        kp[:, 0] = 0
    elif pad == "all_but_one":
        kp = torch.ones(B, T, dtype=torch.uint8, device="cuda")
        kp[torch.arange(B), torch.arange(B) % T] = 0
    if kp is not None:                    # NaN in every padded row: must reach no output
        kv.view(B, T, -1)[kp.bool()] = float("nan")
    dout = torch.randn(B, d, device="cuda", generator=g).bfloat16()
    return kv, q, kp, dout


CASES = []
_BS = [1, 4, 8, 64]
_PADS = [None, "ragged", "all_but_one"]
for i, T in enumerate([1, 2, 15, 16, 196, 256, 750, 1023]):
    for j, (d, H) in enumerate([(256, 4), (1536, 24)]):
        B = _BS[(i + j) % 4]
        if d == 1536 and T >= 750 and B == 64:
            B = 8
        CASES.append((B, T, d, _PADS[(i + 2 * j) % 3], "init" if (i + j) % 2 == 0 else "peaky"))
CASES += [(64, 196, 256, "ragged", "peaky"), (8, 750, 1536, "ragged", "init"), (4, 1, 1536, "all_but_one", "peaky")]


@pytest.mark.parametrize("B,T,d,pad,q_scale", CASES)
def test_attn_pool_forward_backward_within_bounds(B, T, d, pad, q_scale):
    need_gpu()
    from one_peace_b200 import kernels as K
    kv, q, kp, dout = _inputs(B, T, d, pad, q_scale, seed=B * 1000 + T)
    out, lse = K.attn_pool_fwd(kv, q, kp, B, T)
    clean = kv.clone()
    if kp is not None:
        clean.view(B, T, -1)[kp.bool()] = 0
    ro, rl, bo, bl = pool_fwd_ref(clean, q, kp, B, T)
    assert torch.isfinite(out).all() and torch.isfinite(lse).all()
    assert excess(out, ro, bo) <= 1, excess(out, ro, bo)
    assert excess(lse, rl, bl) <= 1
    dkv, dq = K.attn_pool_bwd(kv, q, kp, lse, dout, B, T)
    rkv, rdq, bkv, bdq = pool_bwd_ref(clean, q, kp, dout, B, T)
    assert torch.isfinite(dkv).all() and torch.isfinite(dq).all()
    assert excess(dkv, rkv, bkv) <= 1, excess(dkv, rkv, bkv)
    assert excess(dq, rdq, bdq) <= 1, excess(dq, rdq, bdq)
    if kp is not None:
        assert (dkv.view(B, T, -1)[kp.bool()] == 0).all()
    out2, lse2 = K.attn_pool_fwd(kv, q, kp, B, T)
    dkv2, dq2 = K.attn_pool_bwd(kv, q, kp, lse, dout, B, T)
    assert torch.equal(out, out2) and torch.equal(lse, lse2) and torch.equal(dkv, dkv2) and torch.equal(dq, dq2)


def test_attn_pool_writes_nothing_outside_outputs():
    need_gpu()
    from one_peace_b200 import _lib
    B, T, d = 4, 33, 256
    H = d // 64
    kv, q, kp, dout = _inputs(B, T, d, "ragged", "peaky", seed=3)
    canvas = torch.full((B * d + 256,), float("nan"), dtype=torch.bfloat16, device="cuda")
    lse_c = torch.full((B * H + 64,), float("nan"), device="cuda")
    lib = _lib.load()
    st = lib.opb_attn_pool_fwd(kv.data_ptr(), q.data_ptr(), kp.data_ptr(), canvas[128:].data_ptr(), lse_c[32:].data_ptr(), B, T, d,
                               torch.cuda.current_stream().cuda_stream)
    assert st == 0
    torch.cuda.synchronize()
    assert canvas[:128].isnan().all() and canvas[128 + B * d:].isnan().all() and not canvas[128:128 + B * d].isnan().any()
    assert lse_c[:32].isnan().all() and lse_c[32 + B * H:].isnan().all()
    lse = lse_c[32:32 + B * H].view(B, H).contiguous()
    dkv_c = torch.full((B * T * 2 * d + 512,), float("nan"), dtype=torch.bfloat16, device="cuda")
    dq_c = torch.full((d + 64,), float("nan"), device="cuda")
    ws = torch.empty(B * d, device="cuda")
    st = lib.opb_attn_pool_bwd(kv.data_ptr(), q.data_ptr(), kp.data_ptr(), lse.data_ptr(), dout.data_ptr(), dkv_c[256:].data_ptr(),
                               ws.data_ptr(), dq_c[32:].data_ptr(), B, T, d, torch.cuda.current_stream().cuda_stream)
    assert st == 0
    torch.cuda.synchronize()
    n = B * T * 2 * d
    assert dkv_c[:256].isnan().all() and dkv_c[256 + n:].isnan().all() and not dkv_c[256:256 + n].isnan().any()
    assert dq_c[:32].isnan().all() and dq_c[32 + d:].isnan().all() and not dq_c[32:32 + d].isnan().any()


def _pad_cols(z, n_pad):
    full = torch.full((z.shape[0], n_pad), float("nan"), device="cuda")        # NaN pad columns: never read
    full[:, :z.shape[1]] = z
    return full


@pytest.mark.parametrize("C", [1, 2, 309, 3129])
@pytest.mark.parametrize("mode", [HARD, SOFT, MULTI])
def test_classify_loss_within_bounds(C, mode):
    need_gpu()
    from one_peace_b200 import kernels as K
    rows = 37
    g = torch.Generator(device="cuda").manual_seed(C * 10 + mode)
    z = 4 * torch.randn(rows, C, device="cuda", generator=g)
    n_pad = (C + 7) // 8 * 8
    zp = _pad_cols(z, n_pad)
    labels = targets = None
    eps = 0.0
    if mode == HARD:
        labels = torch.randint(0, C, (rows,), device="cuda", generator=g)
        labels[3] = -100                                        # ignore_index row
        eps = 0.1
    elif mode == SOFT:
        targets = torch.softmax(torch.randn(rows, C, device="cuda", generator=g), 1)
    else:
        targets = (torch.rand(rows, C, device="cuda", generator=g) < 0.3).float()
    tk = _pad_cols(targets, n_pad) if targets is not None else None
    row_loss, dl, corr, out2 = K.classify_loss(zp, C, mode, labels=labels, targets=tk, eps=eps)
    r = loss_ref(z, C, mode, labels=labels, targets=targets, eps=eps)
    assert excess(row_loss, r["row_loss"], r["b_row_loss"]) <= 1
    assert excess(dl[:, :C], r["dlogits"], r["b_dlogits"]) <= 1
    assert (dl[:, C:] == 0).all()
    assert excess(corr, r["row_correct"], r["b_row_correct"]) <= 1
    assert excess(out2[0], r["loss"], r["b_loss"]) <= 1
    assert excess(out2[1], r["n_correct"], r["b_n_correct"]) <= 1
    again = K.classify_loss(zp, C, mode, labels=labels, targets=tk, eps=eps)
    assert all(torch.equal(a, b) for a, b in zip((row_loss, dl, corr, out2), again))


def test_hinge_loss_within_bounds():
    need_gpu()
    from one_peace_b200 import kernels as K
    G, nc = 64, 4
    g = torch.Generator(device="cuda").manual_seed(9)
    z = torch.randn(G * nc, 1, device="cuda", generator=g)
    zp = _pad_cols(z, 8)
    labels = torch.randint(0, nc, (G,), device="cuda", generator=g)
    row_loss, dl, corr, out2 = K.classify_loss(zp, 1, HINGE, labels=labels, num_choices=nc)
    r = loss_ref(z, 1, HINGE, labels=labels, num_choices=nc)
    assert excess(row_loss, r["row_loss"], r["b_row_loss"]) <= 1
    assert torch.equal(dl[:, :1].double(), r["dlogits"]) and (dl[:, 1:] == 0).all()
    assert torch.equal(corr.double(), r["row_correct"])
    assert excess(out2[0], r["loss"], r["b_loss"]) <= 1 and out2[1].item() == r["n_correct"].item()
    # hinge_loss.py:52 in torch (ties aside, its gradient is the kernel's)
    zt = z.detach().double().view(G, nc).requires_grad_(True)
    ref = torch.max(torch.tensor(0.0, device="cuda", dtype=torch.float64), 1 + zt - zt.gather(1, labels[:, None])).sum()
    ref.backward()
    assert math.isclose(out2[0].item(), ref.item(), rel_tol=1e-5)
    assert torch.allclose(dl[:, 0].double().view(G, nc), zt.grad)
