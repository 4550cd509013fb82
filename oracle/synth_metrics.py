"""TEST INFRASTRUCTURE.  Seeded evaluation streams of the classification metrics (metrics/accuracy.py, metrics/map.py), shared by
the golden-vector generator (oracle/make_golden_metrics.py), the metric tests and scripts/bench_eval_metrics.py.  Everything
is drawn from seeded CPU generators in a fixed order; the fixture keeps only what the reference returned."""
import torch

# name -> (rows n, classes C, target kind, logits dtype, batch cuts as fractions of n)
#   hard: int64 labels; hard_f32: fp32 labels (compared as torch.eq promotes); soft: VQA-style scores in {0, 0.3, 0.6, 0.9, 1};
#   aqa: AQA's eval_step view, [4B, 1] logits of rows padded to 8 columns reshaped into [B, 4] (row stride 32, column stride 8)
ACC_CASES = {
    "c1": (37, 1, "hard", torch.float32),
    "nlvr2_c2_bf16": (300, 2, "hard", torch.bfloat16),
    "c4_f32_labels": (257, 4, "hard_f32", torch.float32),
    "vggsound_c309": (500, 309, "hard", torch.float32),
    "vqa_c3129_soft": (96, 3129, "soft", torch.float32),
    "c3129_bf16": (64, 3129, "hard", torch.bfloat16),
    "aqa_view": (50, 4, "aqa", torch.float32),
}

# name -> (rows N, classes C, logits dtype, batch size of the evaluation stream)
MAP_CASES = {
    "fsd50k_bf16": (2003, 200, torch.bfloat16, 8),
    "batches_f32": (333, 200, torch.float32, 50),
}

# the column kinds of a MAP case, in this order (the rest of the columns are "general")
MAP_SPECIAL = ("saturated",) * 20 + ("no_positive", "all_equal", "dense") + ("sparse",) * 27


def batch_cuts(n, seed):
    """Uneven batch boundaries 0 = c0 < c1 < ... = n: a one-row batch, a short one and random sizes."""
    g = torch.Generator().manual_seed(seed)
    cuts = [0, 1, min(7, n)]
    while cuts[-1] < n:
        cuts.append(min(n, cuts[-1] + int(torch.randint(5, 97, (1,), generator=g))))
    return sorted(set(cuts))


def accuracy_case(name, seed=0):
    """-> (ids int64 [n], logits [n, C] (a strided view for 'aqa'), targets, cuts).  A third of the rows are quantised to
    halves so that argmax ties are common; some rows hold one NaN, two NaNs or only NaNs."""
    n, C, kind, dtype = ACC_CASES[name]
    g = torch.Generator().manual_seed(7000 + seed + sum(map(ord, name)))
    if kind == "aqa":
        B = n
        padded = torch.full((4 * B, 8), 123.0)                 # autograd_classify's rows padded to a multiple of 8 columns
        padded[:, :1] = torch.randn(4 * B, 1, generator=g)
        padded[::3, :1] = torch.round(padded[::3, :1])
        logits = padded[:, :1].reshape(B, 4)                   # view: strides (32, 8)
        assert logits.stride() == (32, 8)
        targets = torch.randint(0, 4, (B,), generator=g)
        ids = torch.randperm(B, generator=g) + 50000
        return ids, logits, targets, batch_cuts(B, seed + 1)
    x = 2.0 * torch.randn(n, C, generator=g)
    q = torch.rand(n, generator=g) < 0.35
    x[q] = torch.round(x[q]) * 0.5
    for r in range(0, n, 11):
        x[r, int(torch.randint(0, C, (1,), generator=g))] = float("nan")
    for r in range(5, n, 23):
        x[r, torch.randint(0, C, (2,), generator=g)] = float("nan")
    x[n - 1] = float("nan")
    if C > 1:
        x[n - 2] = float("-inf")
        x[n - 3, :] = 0.0
        x[n - 3, C // 2] = -0.0
    logits = x.to(dtype)
    if kind == "soft":
        targets = torch.zeros(n, C)
        k = torch.randint(1, 4, (n,), generator=g)
        vals = torch.tensor([0.3, 0.6, 0.9, 1.0])
        for r in range(n):
            cols = torch.randint(0, C, (int(k[r]),), generator=g)
            targets[r, cols] = vals[torch.randint(0, 4, (int(k[r]),), generator=g)]
            if r % 4 == 0:                                     # the argmax itself scores
                targets[r, int(torch.nan_to_num(logits[r].float(), nan=float("inf")).argmax())] = 0.9
    else:
        targets = torch.randint(0, C, (n,), generator=g)
        hit = torch.rand(n, generator=g) < 0.5                 # half the rows hit (where the argmax is a real index)
        am = logits.float().argmax(1)
        targets[hit] = am[hit]
        if kind == "hard_f32":
            targets = targets.float()
    ids = torch.randperm(n, generator=g) + 1000
    return ids, logits, targets, batch_cuts(n, seed)


def map_case(name, seed=0):
    """-> (ids int64 [N], logits [N, C], multi-hot targets fp32 [N, C], cuts every batch size rows, the last one shorter) with
    column kinds: 'general' (logits ~ 1.5 z + shift in [-12, 8] with labels drawn from a logistic of the logit, so AP is
    neither 0 nor 1), 'saturated' (|x| in [17, 40]: distinct logits above 16.6 share p = 1.0f), 'no_positive', 'all_equal',
    'dense' (90 % positive) and 'sparse' (1 to 3 positives).  bf16 logits make many ties in every column.  No logit lies in
    (8, 17), where fp32 sigmoids that differ by an ulp or two could merge different neighbours into one probability, so every
    such sigmoid (torch's CUDA one, the fixture's stand-in) gives the same tie groups."""
    N, C, dtype, bs = MAP_CASES[name]
    g = torch.Generator().manual_seed(9000 + seed + sum(map(ord, name)))
    kinds = ["general"] * (C - len(MAP_SPECIAL)) + list(MAP_SPECIAL)
    x = torch.empty(N, C)
    y = torch.zeros(N, C)
    for c, kind in enumerate(kinds):
        if kind == "general":
            x[:, c] = (1.5 * torch.randn(N, generator=g) + 2.0 * torch.rand(1, generator=g) - 3.0).clamp(-12.0, 8.0)
            y[:, c] = (torch.rand(N, generator=g) < torch.sigmoid(x[:, c] + 0.5 * torch.randn(N, generator=g))).float()
        elif kind == "saturated":
            s = torch.where(torch.rand(N, generator=g) < 0.6, 1.0, -1.0)
            x[:, c] = s * (17.0 + 23.0 * torch.rand(N, generator=g))
            y[:, c] = (torch.rand(N, generator=g) < torch.where(s > 0, 0.7, 0.2)).float()
        elif kind == "no_positive":
            x[:, c] = torch.randn(N, generator=g)
        elif kind == "all_equal":
            x[:, c] = 0.25
            y[:, c] = (torch.rand(N, generator=g) < 0.3).float()
        elif kind == "dense":
            x[:, c] = torch.randn(N, generator=g)
            y[:, c] = (torch.rand(N, generator=g) < 0.9).float()
        else:
            x[:, c] = torch.randn(N, generator=g) - 2.0
            y[torch.randint(0, N, (int(torch.randint(1, 4, (1,), generator=g)),), generator=g), c] = 1.0
    logits = x.to(dtype)
    ids = torch.randperm(N, generator=g) + 20000
    cuts = list(range(0, N, bs)) + [N]
    return ids, logits, y, cuts
