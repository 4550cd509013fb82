"""fairseq ``--user-dir`` hook (reference: one_peace/user_module/__init__.py:1-7): importing this package fires
the @register_model / @register_criterion / @register_optimizer decorators of the sm_90a replacements, which
register under the reference's own names (one_peace_retrieval, one_peace_pretrain, one_peace_classify,
image_text_retrieval_criterion, audio_text_retrieval_criterion, image_text_pretrain_loss, audio_text_pretrain_loss,
classify_criterion, hinge_loss, refcoco_criterion, adjust_adam).  See INTEGRATION.md."""
from .. import criterions, optim  # noqa: F401
from ..one_peace import one_peace_classify, one_peace_pretrain, one_peace_retrieval  # noqa: F401
