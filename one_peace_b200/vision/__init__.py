"""The vision branch's ImageNet classifier (one_peace_vision/classification): ``models_vit`` and the criteria of ``main_ft.py``."""
