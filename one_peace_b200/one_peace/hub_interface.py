"""Drop-in for the embedding API of models/one_peace/hub_interface.py:53-225.

``from_pretrained`` / ``OnePeaceHubInterface.extract_{text,image,audio}_features`` keep the reference
signatures.  Pre-processing (BPE, image transforms, audio loading) stays Python in the reference and is not
part of the accelerated path: ``process_*`` delegate to user-supplied callables.
"""
import torch

from .one_peace_classify import OnePeaceClassifyConfig, OnePeaceClassifyModel
from .one_peace_pretrain import OnePeacePretrainConfig, OnePeacePretrainModel
from .one_peace_retrieval import OnePeaceRetrievalConfig, OnePeaceRetrievalModel
from ..unify_model_config import one_peace_4b_decoder_config, one_peace_4b_encoder_config


class _Dictionary:
    """Minimal stand-in for fairseq's Dictionary: the model only needs len() and pad() (adapter/text.py:41-43).
    50,264 = 4 specials + 50,260 BPE symbols (utils/BPE/dict.txt)."""

    def __init__(self, n=50264, pad=1):
        self._n, self._pad = n, pad

    def __len__(self):
        return self._n

    def pad(self):
        return self._pad


def from_pretrained(model_name_or_path=None, model_type="one_peace_retrieval", device="cuda", dtype="float32",
                    state_dict=None, head_type="val", layers=40, embed_dim=1536, ffn_embed_dim=6144,
                    attention_heads=24, patch_image_size=256, vocab_size=50264, decoder=None, use_audio=None, use_image=True,
                    stage2_pretrain=False, num_classes=None, use_two_images=False, use_pooler=False, head_scale_ratio=1,
                    use_image_features=False):
    """hub_interface.py:53-73.  Loads ``one-peace.pt``-style state dicts (same parameter names, strict except for
    pretraining-only keys) into the sm_90a model.  ``model_name_or_path`` may be a torch checkpoint whose
    'model' entry is the state dict (fairseq layout) or a bare state dict; alternatively pass ``state_dict``.
    model_type="one_peace_classify": the attention-pooling classification model of the fine-tuning recipes (head_type one of
    text / image / audio / vl / al, `num_classes` outputs); its extract_* methods return the logits."""
    if model_type == "one_peace_pretrain":
        # models/one_peace/one_peace_pretrain.py: encoder + lightweight decoder (pretrain_vl_3B.yaml:92-168); `decoder` =
        # dict(embed_dim=, ffn_embed_dim=, layers=, attention_heads=) or None for the 4B recipe's 768 / 2048 / 2 / 12
        # use_audio / use_image=False / stage2_pretrain: the audio-text recipe (pretrain_al_3B.yaml:91,125-127,165-167)
        cfg = OnePeacePretrainConfig()
        cfg.stage2_pretrain = bool(stage2_pretrain)
        cfg.encoder = one_peace_4b_encoder_config(layers, embed_dim, ffn_embed_dim, attention_heads, patch_image_size)
        cfg.encoder.image_adapter.bucket_size = patch_image_size // 16
        cfg.decoder = one_peace_4b_decoder_config(patch_image_size=patch_image_size, **(decoder or {}))
        cfg.encoder.use_audio_moe = cfg.decoder.use_audio_moe = bool(use_audio)
        cfg.encoder.use_image_moe = cfg.decoder.use_image_moe = bool(use_image)
        with torch.device(device):
            model = OnePeacePretrainModel(cfg, _Dictionary(vocab_size))
    elif model_type == "one_peace_retrieval":
        cfg = OnePeaceRetrievalConfig()
        cfg.encoder = one_peace_4b_encoder_config(layers, embed_dim, ffn_embed_dim, attention_heads, patch_image_size)
        with torch.device(device):
            model = OnePeaceRetrievalModel(cfg, _Dictionary(vocab_size), head_type)
    elif model_type == "one_peace_classify":
        cfg = OnePeaceClassifyConfig(attn_pooling=True, use_pooler=bool(use_pooler), head_scale_ratio=head_scale_ratio,
                                     use_image_features=bool(use_image_features))
        cfg.encoder = one_peace_4b_encoder_config(layers, embed_dim, ffn_embed_dim, attention_heads, patch_image_size)
        if num_classes is None:
            raise ValueError("model_type='one_peace_classify' needs num_classes")
        with torch.device(device):
            model = OnePeaceClassifyModel(cfg, _Dictionary(vocab_size), head_type, num_classes, use_two_images)
    else:
        raise NotImplementedError("model_type must be one_peace_retrieval, one_peace_pretrain or one_peace_classify")
    if state_dict is None and model_name_or_path is not None:
        ckpt = torch.load(model_name_or_path, map_location="cpu")
        state_dict = ckpt.get("model", ckpt)
    if state_dict is not None:
        sd = dict(state_dict)
        model.upgrade_state_dict_named(sd, "")
        if model_type == "one_peace_classify":
            sd.pop("logit_scale", None)           # the contrastive temperature of the retrieval / pretraining checkpoints
        model.load_state_dict(sd, strict=True)
    model = model.to({"float32": torch.float32, "fp32": torch.float32, "bfloat16": torch.bfloat16,
                      "bf16": torch.bfloat16}[dtype] if isinstance(dtype, str) else dtype)
    model.eval()
    return OnePeaceHubInterface(model, device=device)


class OnePeaceHubInterface:
    def __init__(self, model, device="cuda", text_tokenizer=None, image_transform=None, audio_loader=None, cuda_graph=False):
        """cuda_graph=True: every (modality, input shape) is captured once into a CUDA graph and replayed afterwards
        (one_peace_b200/graphs.py) — the small-batch embedding API is launch-bound otherwise (212 launches per forward)."""
        self.model = model
        self.device = torch.device(device)
        self._tok, self._img, self._aud = text_tokenizer, image_transform, audio_loader
        self.cuda_graph = cuda_graph
        self._graphs = {}

    def _forward(self, encoder_type, **inputs):
        if not self.cuda_graph:
            return self.model(encoder_type=encoder_type, **inputs)
        from ..graphs import GraphedForward
        key = (encoder_type,) + tuple((k, tuple(v.shape), v.dtype) for k, v in sorted(inputs.items()))
        g = self._graphs.get(key)
        if g is None:
            g = self._graphs[key] = GraphedForward(lambda **kw: self.model(encoder_type=encoder_type, **kw), inputs)
        return g(**inputs)

    # -- pre-processing stays Python (hub_interface.py:134-210) --
    def process_text(self, text_list):
        if self._tok is None:
            raise RuntimeError("pass text_tokenizer= (GPT-2 BPE -> int64 ids, eos appended, pad=1) to the interface")
        return self._tok(text_list).to(self.device)

    def process_image(self, image_list):
        if self._img is None:
            raise RuntimeError("pass image_transform= (resize + CLIP mean/std normalise) to the interface")
        return self._img(image_list).to(self.device)

    def process_audio(self, audio_list):
        if self._aud is None:
            raise RuntimeError("pass audio_loader= (16 kHz mono, per-clip layer-norm, padding mask) to the interface")
        a, m = self._aud(audio_list)
        return a.to(self.device), m.to(self.device)

    def _to_device(self, t):
        if t is None or t.is_cuda:
            return t
        return t.to(self.device, non_blocking=True)

    def _finish(self, feats, out):
        if out is not None:
            out.copy_(feats, non_blocking=True)
            return out
        return feats

    # -- the accelerated path (hub_interface.py:212-222) --
    def _classify(self, **inputs):
        """one_peace_classify: the logits (the reference's extract_text_features drops them; they are returned here)."""
        return self.model(**{k: self._to_device(v) for k, v in inputs.items()})

    def _is_classify(self):
        return isinstance(self.model, OnePeaceClassifyModel)

    @torch.no_grad()
    def extract_text_features(self, src_tokens, out=None):
        if self._is_classify():
            return self._finish(self._classify(src_tokens=src_tokens), out)
        return self._finish(self._forward("text", src_tokens=self._to_device(src_tokens)), out)

    @torch.no_grad()
    def extract_image_features(self, src_images, out=None):
        if self._is_classify():
            return self._finish(self._classify(src_images=src_images), out)
        return self._finish(self._forward("image", src_images=self._to_device(src_images)), out)

    @torch.no_grad()
    def extract_audio_features(self, src_audios, audio_padding_masks, out=None):
        if self._is_classify():
            return self._finish(self._classify(src_audios=src_audios, audio_padding_masks=audio_padding_masks), out)
        return self._finish(self._forward("audio", src_audios=self._to_device(src_audios),
                                          audio_padding_masks=self._to_device(audio_padding_masks)), out)

    @torch.no_grad()
    def extract_vl_features(self, src_images, src_tokens, out=None):
        """one_peace_classify with head_type 'vl' (hub_interface.py:224-225): the logits of an image-text pair."""
        if not self._is_classify():
            raise NotImplementedError("extract_vl_features needs model_type='one_peace_classify'")
        return self._finish(self._classify(src_images=src_images, src_tokens=src_tokens), out)
