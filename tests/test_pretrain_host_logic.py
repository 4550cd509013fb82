"""CPU: host-side index logic of the pretraining path (no kernels): modality-major <-> batch-major row permutations, the
decoder canvas index, preserve-id flattening and the DCL row selections, against the oracle's torch restatement of the
reference lines they replace."""
import torch

import restated as R
import synth


def test_seq_layout_permutations_are_inverse_and_ordered():
    from one_peace_b200.autograd import SeqLayout
    B, parts = 3, [("text", 5), ("image", 7)]
    lay = SeqLayout(B, parts, "cpu")
    assert lay.S == 12 and lay.M == 36 and lay.offs == [0, 15] and lay.los == [0, 5]
    x_mm = torch.arange(lay.M).float()[:, None]
    x_bm = x_mm[lay.to_bm]
    assert torch.equal(x_bm[lay.to_mm], x_mm)                            # inverse permutations
    # batch-major = torch.cat([text (B,5), image (B,7)], dim=1) of the modality-major blocks (transformer_encoder.py:127-134)
    want = torch.cat([x_mm[:15].view(B, 5, 1), x_mm[15:].view(B, 7, 1)], dim=1).reshape(-1, 1)
    assert torch.equal(x_bm, want)
    rs = lay.row_scale(torch.tensor([1.0, 0.0, 2.0]))
    assert torch.equal(rs[:15].view(B, 5)[:, 0], torch.tensor([1.0, 0.0, 2.0])) and torch.equal(rs[15:].view(B, 7)[:, 3], torch.tensor([1.0, 0.0, 2.0]))
    single = SeqLayout(2, [("text", 4)], "cpu")
    assert single.to_bm is None and single.to_mm is None


def test_canvas_index_and_flat_ids_match_the_reference_scatter():
    from one_peace_b200.adapter.text import canvas_index, flat_ids
    g = torch.Generator().manual_seed(0)
    B, S, Kk, d = 3, 9, 5, 4
    ids = torch.stack([torch.randperm(S, generator=g)[:Kk].sort().values for _ in range(B)])
    ids[1, -2:] = -1
    emb = torch.randn(B, Kk, d, generator=g)
    mask_token = torch.randn(1, d, generator=g)
    want = R.canvas(ids, emb, mask_token, S)                             # adapter/text.py:135-142
    idx = canvas_index(ids, S)
    got = torch.where((idx >= 0)[:, None], emb.reshape(-1, d)[idx.clamp_min(0)], mask_token.expand(B * S, -1)).view(B, S, d)
    assert torch.equal(got, want)
    full = torch.randn(B, S, d, generator=g)
    fi = flat_ids(ids, S)
    gathered = torch.where((fi >= 0)[:, None], full.reshape(-1, d)[fi.clamp_min(0)], torch.zeros(1, d)).view(B, Kk, d)
    pid = ids.masked_fill(ids.eq(-1), Kk - 1)
    ref = full.gather(1, pid[:, :, None].expand(-1, -1, d)) * (~ids.eq(-1))[:, :, None]      # padded rows are zeroed by the encoder
    assert torch.equal(gathered, ref)


def test_dcl_indices_select_the_reference_rows():
    """Masked, non-padded, non-CLS student rows first; then every other non-padded non-CLS teacher row
    (image_text_pretrain_loss.py:190-202; the soft-max is invariant to the column order)."""
    from one_peace_b200.autograd_general import dcl_indices
    sample = synth.pretrain_sample(seed=3)
    ni = sample["net_input"]
    mask, pm = ni["text_mask_indices"], ni["src_tokens"].eq(1)
    stu, tea = dcl_indices(mask, pm)
    B, S = mask.shape
    d = 8
    g = torch.Generator().manual_seed(1)
    student = torch.randn(B, S, d, generator=g)
    teacher = torch.randn(B, S, d, generator=g)
    want = R.dcl_loss(student, teacher, mask, pm, 2.5, 0.1)
    s_rows = torch.nn.functional.normalize(student.reshape(-1, d)[stu], dim=1)
    t_rows = torch.nn.functional.normalize(teacher.reshape(-1, d)[tea], dim=1)
    lp = torch.log_softmax(2.5 * s_rows @ t_rows.t(), -1)
    got = R.label_smoothed_nll(lp, torch.arange(stu.numel()), 0.1)
    torch.testing.assert_close(got, want, atol=1e-6, rtol=1e-6)
    stu_i, tea_i = dcl_indices(ni["image_mask_indices"], None)
    assert stu_i.numel() == int(ni["image_mask_indices"][:, 1:].sum()) and tea_i.numel() == B * (ni["image_mask_indices"].shape[1] - 1)


def test_pretrain_model_parameter_names_match_the_reference(golden_dir):
    import os
    from one_peace_b200.one_peace.hub_interface import from_pretrained
    T = synth.PRETRAIN_TINY
    fx = torch.load(os.path.join(golden_dir, "pretrain_criterion.pt"), weights_only=False)
    sd = synth.make_pretrain_state_dict(**T, seed=0)
    model = from_pretrained(state_dict=sd, model_type="one_peace_pretrain", layers=T["layers"], embed_dim=T["embed_dim"],
                            ffn_embed_dim=T["ffn"], attention_heads=T["heads"], patch_image_size=T["res"], vocab_size=T["vocab"],
                            decoder=dict(embed_dim=T["dec_dim"], ffn_embed_dim=T["dec_ffn"], layers=T["dec_layers"],
                                         attention_heads=T["dec_heads"]), device="cpu").model
    own = {n: tuple(p.shape) for n, p in model.named_parameters()}
    for name, summ in fx["grads"].items():                    # names / shapes recorded from the reference's own model
        assert name in own and own[name] == tuple(summ["shape"]), name
    assert set(own) == set(fx["grads"]) | {n for n in own if n not in fx["grads"]}
    missing = [n for n in own if n not in sd]
    assert not missing, missing                               # strict load consumed the reference-layout state dict
