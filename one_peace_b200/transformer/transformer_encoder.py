"""Drop-in for ``TransformerEncoder`` (models/transformer/transformer_encoder.py:23-251).

Same constructor, same parameter names (layers.N.*, {text,image,audio}_layer_norm).  ``forward`` keeps
the reference signature (text_info / image_info / audio_info tuples from the adapters + encoder_type);
the tuples carry the fp32 residual stream (B,S,d), a uint8/bool padding mask (or None) and the
batch-shared (H,S,S_pad) bias table instead of the reference's expanded (B,H,S,S) tensor.
"""
import torch
import torch.nn as nn

from .. import kernels as K
from ..autograd import _pick
from ..components import LayerNorm, PackCache, f32
from ..fairseq_compat import FairseqEncoder
from .transformer_layer import TransformerEncoderLayer


class TransformerEncoder(FairseqEncoder):
    def __init__(self, cfg, dictionary, use_text_norm, use_image_norm, use_audio_norm):
        self.cfg = cfg
        super().__init__(dictionary)
        self.register_buffer("version", torch.Tensor([3]))
        if cfg.layerdrop > 0.0:
            raise NotImplementedError("layerdrop is 0 in every ONE-PEACE config")
        self.max_positions = cfg.max_positions
        self.num_attention_heads = cfg.attention_heads
        dpr = [x.item() for x in torch.linspace(0, cfg.drop_path_rate, cfg.layers)]
        self.layers = nn.ModuleList([TransformerEncoderLayer(cfg, drop_path_rate=dpr[i]) for i in range(cfg.layers)])
        self.num_layers = len(self.layers)
        self.text_layer_norm = LayerNorm(cfg.embed_dim) if (cfg.use_text_moe and use_text_norm) else None
        self.image_layer_norm = LayerNorm(cfg.embed_dim) if (cfg.use_image_moe and use_image_norm) else None
        self.audio_layer_norm = LayerNorm(cfg.embed_dim) if (cfg.use_audio_moe and use_audio_norm) else None
        self._cache = PackCache()

    def final_norm_pack(self, modality):
        ln = getattr(self, f"{modality}_layer_norm")
        if ln is None:
            return None
        return f32(ln.weight), f32(ln.bias), ln.eps

    def run_layers(self, info, encoder_type):
        """Runs the 40-layer hot loop in place on the residual stream; returns (x [B,S,d] fp32, pad)."""
        if encoder_type not in ("text", "image", "audio"):
            # 'vl' / 'al' (concatenated sequences with per-modality FFN) belong to the pretraining path
            raise NotImplementedError(f"encoder_type={encoder_type!r}: only single-modality encoders are built")
        for layer in self.layers:
            layer.check_structure()
        x, pad, bias_list = info
        B, S, d = x.shape
        x = x.contiguous()
        key_pad = None
        if pad is not None:
            key_pad = pad.to(torch.uint8).contiguous()
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.layers.parameters())):
            # training: hand-written backward behind torch.autograd (one_peace_b200/autograd.py); bias_list holds dense
            # (H,S,S_pad) tensors here
            from ..autograd import run_encoder_stack
            return run_encoder_stack(self, x, bias_list, key_pad, encoder_type), pad
        self.run_fused(x.view(B * S, d), bias_list, key_pad, B, S, encoder_type)
        return x, pad

    def run_fused(self, rows, biases, key_pad, B, S, modality, inputs=None):
        """The fused-LayerNorm layer loop (TransformerEncoderLayer.forward_rows_fused) of a single-modality sequence.
        rows: fp32 [B*S, d] residual stream, updated in place and returned.  biases: 0, 1 or L kernels.RelPosBias.
        inputs: None, or a list to which a copy of each layer's input rows is appended (the recompute backward of
        autograd.EncoderStackFn starts from them)."""
        ws = TransformerEncoderLayer.fused_workspace(B * S, rows.shape[1], self.cfg.ffn_embed_dim, self.num_attention_heads,
                                                     rows.device)
        K.row_stats_cast(rows, ws["xb"], ws["mu"], ws["rstd"], eps=self.layers[0].self_attn_layer_norm.eps)
        ln1 = dict(ln_mu=ws["mu"], ln_rstd=ws["rstd"])
        for i, layer in enumerate(self.layers):
            if inputs is not None:
                inputs.append(rows.clone())
            ln1 = layer.forward_rows_fused(rows, ws["xb"], ln1, ws, _pick(biases, i), key_pad, B, S, modality)
        return rows

    def forward_general(self, parts):
        """General encoder forward (transformer_encoder.py:73-232) for concatenated modalities ('vl' / 'al'), preserve_ids
        student passes and the decoder.  parts = [(modality, x fp32 (B,S_p,d), pad uint8 (B,S_p) or None, bias source or None)]
        in sequence order.  Returns ([features fp32 (B,S_p,d) per part, after that modality's final LayerNorm], [pad per part]).
        Differentiable end to end (one_peace_b200/autograd.py, autograd_general.py)."""
        from ..autograd import SeqLayout, run_general_stack
        from ..autograd_general import BlockBiasFn, FinalNormFn, ZeroPadFn
        B, d = parts[0][1].shape[0], parts[0][1].shape[2]
        dev = parts[0][1].device
        H = self.num_attention_heads
        lay = SeqLayout(B, [(m, x.shape[1]) for m, x, _, _ in parts], dev)
        x_mm = torch.cat([x.reshape(-1, d) for _, x, _, _ in parts], dim=0) if len(parts) > 1 else parts[0][1].reshape(-1, d)
        pads = [p.to(torch.uint8) if p is not None else torch.zeros(B, x.shape[1], dtype=torch.uint8, device=dev)
                for _, x, p, _ in parts]
        any_pad = any(p is not None for _, _, p, _ in parts)
        if any_pad:                                               # x * (1 - padding_mask), :139-142
            x_mm = ZeroPadFn.apply(x_mm, torch.cat([p.reshape(-1) for p in pads]).contiguous())
        srcs = [(pi, bs) for pi, (_, _, _, bs) in enumerate(parts) if bs is not None]
        biases = []
        if srcs:                                                  # :144-162: per-modality diagonal blocks of one canvas per table
            n_tab = len(srcs[0][1]["tables"])
            for j in range(n_tab):
                blocks = tuple((bs["bucket"], bs["ids"], bs["n"], lay.los[pi]) for pi, bs in srcs)
                biases.append(BlockBiasFn.apply((H, lay.S, blocks), *[bs["tables"][j] for _, bs in srcs]))
        # padded keys are excluded only through the bias (-inf fill, :159-160): without a bias they are attended
        key_pad = torch.cat(pads, dim=1).contiguous() if (any_pad and biases) else None
        need_grad = torch.is_grad_enabled() and (x_mm.requires_grad or any(q.requires_grad for q in self.parameters()))
        out = run_general_stack(self, x_mm.to(torch.float32), lay, key_pad, biases, need_grad)
        feats = []
        for pi, (m, x, _, _) in enumerate(parts):
            ln = getattr(self, f"{m}_layer_norm")
            rows = out[lay.rows(pi)]
            if ln is not None:
                rows = FinalNormFn.apply(rows, ln.weight, ln.bias, ln.eps)
            feats.append(rows.view(B, x.shape[1], d))
        return feats, [p if p is not None else None for _, _, p, _ in parts]

    def forward(self, text_info, image_info, audio_info, return_all_hiddens: bool = False, encoder_type=None):
        if return_all_hiddens:
            raise NotImplementedError("return_all_hiddens is only used by the segmentation/detection heads")
        info = {"text": text_info, "image": image_info, "audio": audio_info}.get(encoder_type)
        x, pad = self.run_layers(info, encoder_type)
        if x.requires_grad:
            raise NotImplementedError("per-token features with gradients (pretraining decoder / DCL path) are not built; "
                                      "the retrieval heads train through OnePeaceRetrievalModel.forward")
        B, S, d = x.shape
        pk = self.final_norm_pack(encoder_type)
        if pk is not None:
            out = torch.empty_like(x)
            K.layernorm(x.view(B * S, d), pk[0], pk[1], out.view(B * S, d), eps=pk[2])
            x = out
        return {"encoder_out": [x.transpose(0, 1)], "encoder_padding_mask": pad, "text_encoder_states": [],
                "image_encoder_states": [], "audio_encoder_states": []}
