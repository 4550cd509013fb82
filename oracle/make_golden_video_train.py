"""TEST INFRASTRUCTURE.  Generates tests/golden/video_train.pt by executing the reference's OWN video backbone
(one_peace_vision/video/mmaction_custom/models/backbones/onepeace.py, under oracle/ref_stub_video.py's stubs) in train mode,
in fp64, on the tiny config oracle/synth_video.VIDEO_TINY with the weights of synth_video.video_state_dict.  It needs
the reference source tree:

    python oracle/make_golden_video_train.py

Stored, for a fixed cotangent of forward()'s output [B, d, T, 1, 1]:
  - "plain": drop_path_rate 0, T = 4, 2 clips: the output and every parameter's gradient;
  - "drop_path": drop_path_rate 0.5 (layer 1 gets p = 0.5, layer 0 p = 0), the same clips: the output, every parameter's
    gradient, and the masks the reference drew.  The module-level drop_path is wrapped: each call's random tensor is
    drawn again from the RNG state saved before it and stored as its per-frame scale floor(keep + r) / keep, in call
    order (per layer: temporal, spatial, MLP adapter).
Gradients of more than 4096 elements are stored as int8 multiples of rms(row) / 4 per row, lzma-compressed (the
others in bf16), which keeps the fixture under 1 MB; a
stored gradient keeps a cosine above 0.997 with its exact value (checked here for every parameter).
"""
import importlib.util
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_stub  # noqa: E402
import ref_stub_video  # noqa: E402
import synth_video as sv  # noqa: E402
from grad_codec import dequantise, quantise  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
SRC = os.path.join(ref_stub.REF_ROOT, "one_peace_vision", "video", "mmaction_custom", "models", "backbones", "onepeace.py")
T, CLIPS = 4, 2


def _load():
    spec = importlib.util.spec_from_file_location("ref_video_onepeace_train", SRC)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def run_case(ov, drop_path_rate, x, cot):
    torch.manual_seed(0)
    m = ov.OnePeaceViT(num_frames=T, **{**sv.VIDEO_TINY, "drop_path_rate": drop_path_rate})
    shapes = {k: tuple(p.shape) for k, p in m.named_parameters()}
    m.load_state_dict(sv.video_state_dict(shapes, dict(m.named_buffers())), strict=True)
    m = m.double().train()
    masks = []
    orig = ov.drop_path

    def recording(xx, drop_prob=0.0, training=False):
        state = torch.get_rng_state()
        out = orig(xx, drop_prob, training)
        if drop_prob > 0 and training:
            with torch.random.fork_rng(devices=[]):
                torch.set_rng_state(state)
                keep = 1 - drop_prob
                r = (keep + torch.rand((1, xx.shape[1], 1), dtype=xx.dtype, device=xx.device)).floor_()
            masks.append((r[0, :, 0] / keep).clone())
        return out
    ov.drop_path = recording
    try:
        torch.manual_seed(4)
        y = m(x)
    finally:
        ov.drop_path = orig
    (y * cot).sum().backward()
    exact = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}
    grads = quantise(exact)
    for k, g in dequantise(grads).items():
        if exact[k].abs().max() > 0:
            c = torch.nn.functional.cosine_similarity(g.flatten(), exact[k].flatten(), dim=0).item()
            assert c > 0.997, (k, c)
    return dict(out=y.detach().float(), grads=grads, masks=[t.float() for t in masks], drop_path_rate=drop_path_rate)


def main():
    ref_stub_video.install()
    ov = _load()
    torch.set_num_threads(8)
    x = sv.video_clips(T, CLIPS, sv.VIDEO_TINY["bucket_size"]).double()
    cot = torch.randn(CLIPS, sv.VIDEO_TINY["embed_dim"], T, 1, 1, generator=torch.Generator().manual_seed(5))
    out = dict(config=dict(sv.VIDEO_TINY), T=T, clips=CLIPS, cot=cot,
               plain=run_case(ov, 0.0, x, cot.double()), drop_path=run_case(ov, 0.5, x, cot.double()))
    assert len(out["plain"]["masks"]) == 0 and len(out["drop_path"]["masks"]) == 3
    path = os.path.join(OUT, "video_train.pt")
    torch.save(out, path)
    print("video_train.pt", os.path.getsize(path), "masks", [m.tolist() for m in out["drop_path"]["masks"]])


if __name__ == "__main__":
    main()
