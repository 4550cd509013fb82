from .recall import Recall  # noqa: F401
from .iou_acc import IouAcc  # noqa: F401
