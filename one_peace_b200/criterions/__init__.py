from .image_text_retrieval_loss import ImageTextRetrievalCriterion  # noqa: F401
from .audio_text_retrieval_loss import AudioTextRetrievalCriterion  # noqa: F401
from .image_text_pretrain_loss import ImageTextPretrainLossCriterion  # noqa: F401
from .audio_text_pretrain_loss import AudioTextPretrainLossCriterion  # noqa: F401
from .classify_loss import ClassifyCriterion  # noqa: F401
from .hinge_loss import HingeLoss  # noqa: F401
from .refcoco_loss import RefCOCOCriterion  # noqa: F401
