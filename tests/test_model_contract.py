"""CPU: the drop-in contract of the model class that does not need a GPU (SURVEY.md 8a/8b) — parameter names and shapes
equal the reference's (checkpoint compatibility, checked against the names recorded from the reference's own modules in
tests/golden/tiny_train_grads.pt), state-dict upgrade / pruning per head type, and the absence of any CPU compute path."""
import os

import pytest
import torch

import synth

TINY = dict(embed_dim=256, ffn=1024, layers=2, heads=4)


def build(head_type, sd=None, device="cpu"):
    from one_peace_b200.one_peace.hub_interface import from_pretrained
    return from_pretrained(state_dict=sd, head_type=head_type, layers=2, embed_dim=256, ffn_embed_dim=1024,
                           attention_heads=4, patch_image_size=224, device=device).model


def test_parameter_names_and_shapes_match_the_reference(golden_dir):
    fx = torch.load(os.path.join(golden_dir, "tiny_train_grads.pt"), weights_only=False)
    sd = synth.make_state_dict(**TINY, seed=0)
    model = build("val", sd)
    own = {n: tuple(p.shape) for n, p in model.named_parameters()}
    for modality in ("text", "image"):
        for name, summ in fx["grads"][modality].items():            # names / shapes recorded from the reference's modules
            assert name in own, name
            assert own[name] == tuple(summ["shape"]), (name, own[name], summ["shape"])
    # every tensor of the synthetic reference-layout state dict was consumed (strict load) and round-trips
    got = model.state_dict()
    for k, v in sd.items():
        assert k in got and tuple(got[k].shape) == tuple(v.shape), k
        assert torch.equal(got[k].float().cpu(), v.float()), k


@pytest.mark.parametrize("head_type,dropped", [("image", ("text_", "audio_")), ("text", ("image_", "audio_")),
                                               ("al", ("image_",)), ("vl", ("audio_",))])
def test_state_dict_is_pruned_per_head_type(head_type, dropped):
    """one_peace_retrieval.py:133-150: keys of modalities the head does not use are dropped before the strict load."""
    sd = synth.make_state_dict(**TINY, seed=1)
    model = build(head_type, sd)
    names = [n for n, _ in model.named_parameters()]
    assert names and not any(any(d in n for d in dropped) for n in names)


def test_forward_without_cuda_fails_loudly():
    model = build("text", synth.make_state_dict(**TINY, modalities=("text",), seed=2))
    tok = torch.randint(4, 1000, (2, 8))
    with torch.no_grad(), pytest.raises(RuntimeError):
        model(src_tokens=tok, encoder_type="text")


def test_unbuilt_layer_structure_raises_in_inference():
    """A layer structure no recipe builds (here scale_fc off) is refused before any kernel runs, as in training."""
    model = build("text", synth.make_state_dict(**TINY, modalities=("text",), seed=2))
    fm = model.encoder_wrapper.fusion_model
    for layer in fm.layers:
        layer.text_ffn[2] = torch.nn.Identity()
    x = torch.randn(2, 8, TINY["embed_dim"])
    with torch.no_grad(), pytest.raises(NotImplementedError):
        fm.run_layers((x, None, None), "text")


def test_adam_chunk_tables_are_cached_by_shape():
    """optim/adam.py `_Table`: the chunk tables of the multi-tensor kernels depend on the tensor SIZES only — a re-allocated .grad
    (new pointer, same shape) must cost one record upload, not a rebuild of the 184 k-chunk tables (that rebuild was 0.3 ms of host
    work per grad-norm call at 1.5 B parameters)."""
    import torch
    from one_peace_b200.optim.adam import _Table
    ps = [torch.zeros(20000), torch.zeros(5)]
    gs = [torch.zeros(20000), torch.zeros(5)]
    tab = _Table()
    ent = lambda grads: [(p, g, g, g, None, 0) for p, g in zip(ps, grads)]
    tab.build(ent(gs), torch.device("cpu"))
    ct, co, n = tab.chunk_tensor, tab.chunk_off, tab.n_chunks
    assert n == -(-20000 // 8192) + 1 and int(ct[-1]) == 1 and int(co[1]) == 8192
    rec0 = tab.tensors.clone()
    tab.build(ent([torch.zeros(20000), torch.zeros(5)]), torch.device("cpu"))          # new gradient tensors, same shapes
    assert tab.chunk_tensor is ct and tab.chunk_off is co                              # tables reused
    assert not torch.equal(tab.tensors, rec0)                                          # records refreshed (new pointers)
    ps.append(torch.zeros(9000))
    tab.build(ent([torch.zeros(20000), torch.zeros(5), torch.zeros(9000)]), torch.device("cpu"))
    assert tab.n_chunks == n + 2 and tab.chunk_tensor is not ct                        # a size change rebuilds them
