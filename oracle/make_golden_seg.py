"""TEST INFRASTRUCTURE.  Generates tests/golden/seg.pt by executing the reference's OWN segmentation backbone
(one_peace_vision/seg/mmseg_custom/models/backbones/onepeace_adapter.py, under oracle/ref_stub_seg.py's stubs) in fp64 on
the CPU.  It needs the reference source tree:

    python oracle/make_golden_seg.py

Stored: the tiny config's key / shape / dtype list; its four output maps for B = 2 seeded images
(synth_seg.seg_images, weights synth_seg.seg_state_dict; sample 0 alone is the B = 1 case, as eval BatchNorm is per
sample); the reference's deform_inputs for that input; the state after init_weights() of a tiny .pkl and a tiny .pth
checkpoint (pos_embed and the shared table on a smaller grid, so both resizes run); and the production config's key list
built on the meta device.
"""
import json
import os
import pickle
import sys
import tempfile
import zlib

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_stub_seg  # noqa: E402
import synth_seg as ss  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "seg.pt")


def _keys(model):
    return [(k, tuple(v.shape), str(v.dtype)) for k, v in model.state_dict().items()]


def _tiny(oa):
    torch.manual_seed(0)
    return oa.OnePeaceAdapter(**ss.SEG_TINY)


def main():
    oa = ref_stub_seg.install()
    am = sys.modules["ref_seg_backbones.adapter_modules"]
    torch.set_num_threads(8)
    m = _tiny(oa)
    out = {"config": dict(ss.SEG_TINY), "keys": _keys(m)}
    m.load_state_dict(ss.seg_state_dict(m), strict=True)
    m = m.double().eval()
    x = ss.seg_images(2, ss.SEG_TINY["bucket_size"])
    with torch.no_grad():
        fs = m(x.double())
    out["maps"] = [f.float().clone() for f in fs]
    d1, d2 = am.deform_inputs(x)
    out["deform_inputs"] = [[t.clone() for t in d1], [t.clone() for t in d2]]
    print("maps", [tuple(f.shape) for f in fs], [f.abs().mean().item() for f in fs])

    # init_weights(): the pretraining layout at a smaller grid (bucket 3 -> 4): pos_embed resized bicubically, the shared
    # table expanded to every layer and resampled by the geometric-sequence interpolation
    g = torch.Generator().manual_seed(3)
    d, heads = ss.SEG_TINY["embed_dim"], ss.SEG_TINY["attention_heads"]
    ckpt = {"image_adapter.pos_embed": torch.randn(3 * 3 + 1, d, generator=g),
            "image_adapter.rel_pos_table_list.0.weight": torch.randn(5 * 5 + 3, heads, generator=g),
            "image_adapter.rp_bucket": torch.zeros(10, 10, dtype=torch.int64),
            "encoder.layers.1.gamma_1": torch.randn(d, generator=g),
            "interactions.0.injector.gamma": torch.randn(d, generator=g),
            "unrelated.weight": torch.randn(3, generator=g)}
    out["pretrained"] = {"ckpt": ckpt}
    with tempfile.TemporaryDirectory() as tmp:
        for ext in ("pkl", "pth"):
            path = os.path.join(tmp, "ckpt." + ext)
            if ext == "pkl":
                with open(path, "wb") as f:
                    pickle.dump({"model": {k: v.clone() for k, v in ckpt.items()}}, f)
            else:
                torch.save({"state_dict": {k: v.clone() for k, v in ckpt.items()}}, path)
            mm = _tiny(oa)
            mm.init_cfg = dict(type="Pretrained", checkpoint=path)
            mm.init_weights()
            st = mm.state_dict()
            keys = ["image_adapter.pos_embed", "encoder.layers.1.gamma_1", "interactions.0.injector.gamma"] + \
                [f"encoder.layers.{i}.rel_pos_table.weight" for i in range(ss.SEG_TINY["layers"])]
            out["pretrained"][ext] = {k: st[k].clone() for k in keys}

    lin = torch.linspace
    torch.linspace = lambda *a, **k: lin(*a, **{**k, "device": "cpu"})
    try:
        with torch.device("meta"):
            big = oa.OnePeaceAdapter(**ss.PRODUCTION)
    finally:
        torch.linspace = lin
    out["production_z"] = zlib.compress(json.dumps(dict(keys=_keys(big))).encode(), 9)
    torch.save(out, OUT)
    print("seg.pt", os.path.getsize(OUT))


if __name__ == "__main__":
    main()
