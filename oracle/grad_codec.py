"""TEST INFRASTRUCTURE.  The storage format of the gradients in tests/golden/video_train.pt
(oracle/make_golden_video_train.py writes it, tests/test_gpu_video_train.py reads it): small tensors in bf16, the others
as int8 multiples of a per-row step, lzma-compressed, so that a fixture of every parameter's gradient stays under 1 MB."""
import lzma

import numpy as np
import torch


def _rows(g):
    return g.reshape(g.shape[0], -1) if g.dim() > 1 else g.reshape(1, -1)


def quantise(grads):
    """{name: fp64 gradient} -> one record: tensors of at most 4096 elements in bf16 ("small"); for the others their
    names, shapes, every row's step rms(row) / 4 (fp32, concatenated) and one lzma blob (a uint8 tensor) of the int8 multiples of it,
    clamped to +-127 steps (32 rms)."""
    small = {k: g.to(torch.bfloat16) for k, g in grads.items() if g.numel() <= 4096}
    big = {k: g for k, g in grads.items() if g.numel() > 4096}
    steps, blobs = [], []
    for g in big.values():
        g2 = _rows(g)
        st = (g2.pow(2).mean(1).sqrt() / 4.0).clamp_min(1e-300)
        steps.append(st)
        blobs.append(torch.round(g2 / st[:, None]).clamp(-127, 127).to(torch.int8).flatten())
    return dict(small=small, names=list(big), shapes=[tuple(g.shape) for g in big.values()], step=torch.cat(steps).float(),
                q=torch.frombuffer(bytearray(lzma.compress(torch.cat(blobs).numpy().tobytes(), preset=9)), dtype=torch.uint8))


def dequantise(rec):
    """-> {name: the stored gradient, fp64}"""
    q = torch.from_numpy(np.frombuffer(lzma.decompress(rec["q"].numpy().tobytes()), dtype=np.int8).copy()).double()
    step = rec["step"].double()
    out, qo, so = {k: g.double() for k, g in rec["small"].items()}, 0, 0
    for name, shape in zip(rec["names"], rec["shapes"]):
        n = torch.Size(shape).numel()
        rows = shape[0] if len(shape) > 1 else 1
        out[name] = (q[qo:qo + n].view(rows, -1) * step[so:so + rows, None]).view(shape)
        qo, so = qo + n, so + rows
    return out
