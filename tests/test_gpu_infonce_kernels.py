"""GPU: the contrastive-head kernels (csrc/infonce.cu and the LSE_PARTIAL / SOFTMAX_GRAD GEMM epilogues) row by row against
the fp64 reference of tests/kernel_ref.py, which starts from the fp32 features: the bf16x3 split, the per-tile partials
and their merge across several column tiles (targets in later tiles, a padded last tile, arg-max ties across tiles), the
ticket-based reduction of infonce_forward over one and two directions, the gradient G . B_hi and d loss / d logit_scale."""
import pytest
import torch

import kernel_ref as R

pytestmark = pytest.mark.gpu
D = 256
SCALE = 12.0


@pytest.fixture(scope="module")
def K():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from one_peace_b200 import kernels
    return kernels


def features(b, n, n_valid, offset, seed, noise=0.8):
    """local rows a, b [b, D] and gathered rows a_all, b_all [n, D] (local rows at `offset`, zero rows from n_valid on)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    nrm = torch.nn.functional.normalize
    n_cls = n_valid or n
    a_all = torch.zeros(n, D, device="cuda")
    b_all = torch.zeros(n, D, device="cuda")
    a_all[:n_cls] = nrm(torch.randn(n_cls, D, device="cuda", generator=g), dim=1)
    b_all[:n_cls] = nrm(a_all[:n_cls] + noise * torch.randn(n_cls, D, device="cuda", generator=g), dim=1)
    return a_all[offset:offset + b].clone(), b_all[offset:offset + b].clone(), a_all, b_all


def splits(K, xa, xb, xa_all, xb_all):
    return K.split_bf16x3([xa, xb, xa_all, xb_all], [0, 0, 1, 1])


def both(a3, b3, a_all3, b_all3):
    return [(a3, b_all3), (b3, a_all3)]


def flat(res):
    """infonce_forward's result as a flat tuple of tensors"""
    return (*res[0], *res[1:])


def test_split_bf16x3_layouts(K):
    """1, 2 and 4 tensors per launch"""
    g = torch.Generator(device="cuda").manual_seed(3)
    xs = [torch.randn(r, D, device="cuda", generator=g) * 10.0 ** torch.empty(r, 1, device="cuda").uniform_(-20, 20, generator=g)
          for r in (37, 200, 800, 3)]
    sides = [0, 1, 1, 0]
    for count in (1, 2, 4):
        outs = K.split_bf16x3(xs[:count], sides[:count])
        for x, side, o in zip(xs, sides, outs):
            hi = x.bfloat16()
            lo = (x - hi.float()).bfloat16()
            want = torch.cat([hi, hi, lo] if side == 0 else [hi, lo, hi], 1)
            assert torch.equal(o.view(torch.int16), want.view(torch.int16)), f"{count} tensor(s)"


def check_direction(K, ref, lse, loss, am, what):
    R.assert_within(lse, ref.lse, ref.dlse, 1.0, torch.float32, what=f"{what} lse")
    R.assert_within(loss, ref.loss, ref.dloss, 1.0, torch.float32, what=f"{what} loss")
    assert int(am.min()) >= 0 and int(am.max()) < ref.n_cls, f"{what}: arg-max outside the classes"
    ok = R.argmax_ok(ref.z, ref.dz, am)
    assert bool(ok.all()), f"{what}: arg-max of rows {ok.logical_not().nonzero().flatten().tolist()} is not a maximum"


@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("n,n_valid", [(800, 0), (800, 789)])
@pytest.mark.parametrize("b", [37, 200, 300])
def test_forward_one_and_two_directions_and_gradient(K, b, n, n_valid, eps):
    """n = 800: four 256-column tiles, the last one partly padding; targets start at column 300 (tile 1 and later)"""
    off = 300
    xa, xb, xa_all, xb_all = features(b, n, n_valid, off, seed=b + n_valid)
    a3, b3, a_all3, b_all3 = splits(K, xa, xb, xa_all, xb_all)
    scale = torch.tensor([SCALE], device="cuda")
    ref_a = R.infonce_ref(xa, xb_all, SCALE, off, eps, n_valid)
    ref_b = R.infonce_ref(xb, xa_all, SCALE, off, eps, n_valid)

    first = K.infonce_forward(both(a3, b3, a_all3, b_all3), scale, off, eps, n_valid=n_valid, rows=True)
    (lse_a, lse_b), out3, loss_ab, am_ab = first
    check_direction(K, ref_a, lse_a, loss_ab[:b], am_ab[:b], "a->b")
    check_direction(K, ref_b, lse_b, loss_ab[b:], am_ab[b:], "b->a")
    tgt = torch.arange(b, device="cuda") + off
    assert out3[1].item() == (am_ab[:b] == tgt).sum().item() and out3[2].item() == (am_ab[b:] == tgt).sum().item()
    mean = (ref_a.loss.sum() + ref_b.loss.sum()) / (2 * b)
    tol = (ref_a.dloss.sum() + ref_b.dloss.sum() + 2.0 ** -16 * (ref_a.loss.abs().sum() + ref_b.loss.abs().sum())) / (2 * b)
    R.assert_within(out3[:1], mean.view(1), tol.view(1), 1.0, torch.float32, what="mean loss")
    again = K.infonce_forward(both(a3, b3, a_all3, b_all3), scale, off, eps, n_valid=n_valid, rows=True)
    for x, y in zip(flat(first), flat(again)):
        assert torch.equal(x, y)

    # one direction: the rows of direction a, bit for bit, and their own mean and hit count
    (lse1,), out1, loss1, am1 = K.infonce_forward([(a3, b_all3)], scale, off, eps, n_valid=n_valid, rows=True)
    check_direction(K, ref_a, lse1, loss1, am1, "one direction")
    assert torch.equal(lse1, lse_a) and torch.equal(loss1, loss_ab[:b]) and torch.equal(am1, am_ab[:b])
    assert out1[1].item() == (am1 == tgt).sum().item() and out1[2].item() == 0
    mean1 = ref_a.loss.sum() / b
    tol1 = (ref_a.dloss.sum() + 2.0 ** -16 * ref_a.loss.abs().sum()) / b
    R.assert_within(out1[:1], mean1.view(1), tol1.view(1), 1.0, torch.float32, what="one-direction mean loss")

    # gradient through the MN-major G . B_all contraction, and d loss / d logit_scale
    coef = 1.0 / (2 * b)
    grad_a, gz_a = K.infonce_grad(a3, b_all3, scale, lse_a, off, eps, D, n_valid=n_valid)
    grad_b, gz_b = K.infonce_grad(b3, a_all3, scale, lse_b, off, eps, D, n_valid=n_valid)
    for ref, grad, xo, what in ((ref_a, grad_a, xb_all, "grad a"), (ref_b, grad_b, xa_all, "grad b")):
        want, tol = R.infonce_grad_ref(ref, xo.bfloat16(), SCALE, coef)
        R.assert_within(grad, want, tol, 1.0, torch.float32, what=what)
    for ref, gz, what in ((ref_a, gz_a, "a"), (ref_b, gz_b, "b")):
        got_rows = gz.view(-1, b).sum(0)
        R.assert_within(got_rows, ref.gz, ref.dgz + 2.0 ** -16 * ref.gz.abs(), 1.0, torch.float32, what=f"sum G z rows {what}")
    ds = K.infonce_dscale(gz_a, gz_b, b, n)
    want = coef * (ref_a.gz.sum() + ref_b.gz.sum())
    tol = coef * (ref_a.dgz.sum() + ref_b.dgz.sum() + 2.0 ** -16 * (ref_a.gz.abs().sum() + ref_b.gz.abs().sum()))
    R.assert_within(ds, want.view(1), tol.view(1), 1.0, torch.float32, what="dscale")


def test_argmax_tie_across_tiles_one_and_two_directions(K):
    """the same gathered row at columns 100 (tile 0) and 300 (tile 1), the best match of local row 5: the lower index wins,
    as torch.argmax picks it"""
    b, n = 37, 512
    xa, xb, xa_all, xb_all = features(b, n, 0, 0, seed=7)
    xb_all[100] = xa[5]
    xb_all[300] = xa[5]
    a3, b3, a_all3, b_all3 = splits(K, xa, xb, xa_all, xb_all)
    scale = torch.tensor([SCALE], device="cuda")
    *_, am_ab = K.infonce_forward(both(a3, b3, a_all3, b_all3), scale, 0, 0.0, rows=True)
    assert am_ab[5].item() == 100
    *_, am1 = K.infonce_forward([(a3, b_all3)], scale, 0, 0.0, rows=True)
    assert am1[5].item() == 100
    z = SCALE * (xa.double() @ xb_all.double().t())
    assert z[5].argmax().item() == 100


def test_forward_ticket_is_reset(K):
    """calls in a row with different b and direction counts (so different grids) give what fresh calls give: the last block
    of each call returns the ticket counter to zero"""
    n, off = 512, 100
    scale = torch.tensor([SCALE], device="cuda")
    calls = [(37, 2), (300, 1), (200, 2), (37, 1), (300, 2)]
    args = {}
    for b in (37, 300, 200):
        xs = features(b, n, 0, off, seed=b)
        args[b] = both(*splits(K, *xs))
    seq = [K.infonce_forward(args[b][:dirs], scale, off, 0.1, rows=True) for b, dirs in calls]
    for (b, dirs), got in zip(calls, seq):
        K._TICKETS.clear()                                  # a fresh zero ticket
        fresh = K.infonce_forward(args[b][:dirs], scale, off, 0.1, rows=True)
        for x, y in zip(flat(got), flat(fresh)):
            assert torch.equal(x, y), f"b = {b}, {dirs} direction(s)"


def test_forward_many_rows(K):
    """b = 3000, one and two directions: many more rows than the reducing block has threads; out3 is the mean of the call's
    own row losses and its hit counts are those of its own arg-max rows"""
    b, n, off = 3000, 3504, 500
    xs = features(b, n, 0, off, seed=11, noise=0.25)
    scale = torch.tensor([SCALE], device="cuda")
    tgt = torch.arange(b, device="cuda", dtype=torch.int32) + off
    for dirs in (1, 2):
        pairs = both(*splits(K, *xs))[:dirs]
        _, out, loss_ab, am_ab = K.infonce_forward(pairs, scale, off, 0.1, rows=True)
        want = loss_ab.double().sum() / (dirs * b)
        R.assert_within(out[:1], want.view(1), want.view(1), R.TAU, torch.float32, what=f"mean loss, {dirs} direction(s)")
        hits = [(am_ab[i * b:(i + 1) * b] == tgt).sum().item() for i in range(dirs)] + [0] * (2 - dirs)
        assert 0 < hits[0] < b, "the inputs should give some hits and some misses"
        assert out[1].item() == hits[0] and out[2].item() == hits[1], f"{dirs} direction(s)"
