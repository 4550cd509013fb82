from .recall import Recall  # noqa: F401
from .iou_acc import IouAcc  # noqa: F401
from .accuracy import Accuracy  # noqa: F401
from .map import MAP  # noqa: F401
