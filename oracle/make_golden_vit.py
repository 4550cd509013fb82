"""TEST INFRASTRUCTURE.  Generates tests/golden/vit.pt by executing the reference's OWN vision classifier
(one_peace_vision/classification/models_vit.py, via oracle/ref_stub.py's timm stub) and its layer-decay rule
(classification/utils/lr_decay.py) on the seeded cases of oracle/synth_vit.py.  It needs the reference source tree:

    python oracle/make_golden_vit.py

Tiny config (2 layers, d = 256, 4 heads, ffn 1024), buckets 4 and 16, both heads, both criteria: logits, loss and every
parameter's grad_summary.  Also the state-dict key / shape / dtype lists of the tiny cases and of the four 4B variants (built
on the meta device), no_weight_decay() and get_layer_id_for_vit of every 4B parameter.  Only the fixture is committed.
"""
import importlib.util
import json
import os
import sys
import zlib

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_stub  # noqa: E402
import synth  # noqa: E402
import synth_vit as sv  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
CLS_DIR = os.path.join(ref_stub.REF_ROOT, "one_peace_vision", "classification")


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _keys(model):
    return [(k, tuple(v.shape), str(v.dtype)) for k, v in model.state_dict().items()]


def _meta_model(mv, variant, **kw):
    """The 4B model on the meta device; the reference reads its drop-path schedule with .item(), so linspace runs on the CPU."""
    lin = torch.linspace
    torch.linspace = lambda *a, **k: lin(*a, **{**k, "device": "cpu"})
    try:
        with torch.device("meta"):
            return getattr(mv, variant)(**kw)
    finally:
        torch.linspace = lin


def vit():
    ref_stub.install()
    mv = _load("ref_models_vit", os.path.join(CLS_DIR, "models_vit.py"))
    lrd = _load("ref_lr_decay", os.path.join(CLS_DIR, "utils", "lr_decay.py"))
    torch.set_num_threads(8)
    out = {"config": dict(sv.VIT_TINY, num_classes=sv.NUM_CLASSES, batch=sv.BATCH), "cases": {}}
    for name, (bucket, pool, crit) in sv.VIT_CASES.items():
        torch.manual_seed(0)
        m = mv.OnePeaceViT(bucket_size=bucket, global_pool=pool, num_classes=sv.NUM_CLASSES, **sv.VIT_TINY)
        shapes = {k: tuple(p.shape) for k, p in m.named_parameters()}
        m.load_state_dict(sv.vit_state_dict(shapes, dict(m.named_buffers())), strict=True)
        img, soft, labels = sv.vit_inputs(bucket)
        m.eval()
        with torch.no_grad():
            logits = m(img)
        m.train()
        m.zero_grad(set_to_none=True)
        loss = sv.criterion(crit, m(img), soft, labels)
        loss.backward()
        out["cases"][name] = dict(keys=_keys(m), logits=logits.clone(), loss=loss.detach().clone(),
                                  grads={n: synth.grad_summary(n, p.grad) for n, p in m.named_parameters() if p.grad is not None})
        print(name, loss.item())
    big = []
    for variant in sv.BIG_VARIANTS:
        for pool in (True, False):
            m = _meta_model(mv, variant, global_pool=pool)
            n_layers = len(m.encoder.layers) + 1
            big.append(dict(variant=variant, pool=pool, keys=_keys(m), no_weight_decay=sorted(m.no_weight_decay()),
                            layer_ids={n: lrd.get_layer_id_for_vit(n, n_layers) for n, _ in m.named_parameters()}))
    # eight near-identical lists of ~860 names: stored as one zlib-compressed JSON document (sv.big_records reads it)
    out["big_z"] = zlib.compress(json.dumps(big).encode(), 9)
    path = os.path.join(OUT, "vit.pt")
    torch.save(out, path)
    print("vit.pt", os.path.getsize(path))


if __name__ == "__main__":
    vit()
