"""Binding to the reference's plugin API (SURVEY.md §8b).

When fairseq is importable the replacement classes subclass fairseq's base classes and register
under the reference's names (so ``--user-dir one_peace_b200/user_module`` swaps them in); when it is not
(this build container, the GPU box) thin shims with the same surface keep the package importable.
"""
import torch.nn as nn

try:  # pragma: no cover - fairseq is not installed in the build image
    from fairseq.models import BaseFairseqModel, FairseqEncoder, register_model
    from fairseq.criterions import FairseqCriterion, register_criterion
    from fairseq.optim import FairseqOptimizer, register_optimizer
    from fairseq.dataclass import FairseqDataclass
    from fairseq import metrics
    HAVE_FAIRSEQ = True
except Exception:  # ImportError or transitive failures (omegaconf, hydra ...)
    HAVE_FAIRSEQ = False

    class BaseFairseqModel(nn.Module):
        def __init__(self):
            super().__init__()

        def set_num_updates(self, num_updates):
            for m in self.modules():
                if hasattr(m, "set_num_updates") and m is not self:
                    m.set_num_updates(num_updates)

        def upgrade_state_dict_named(self, state_dict, name):
            pass

    class FairseqEncoder(nn.Module):
        def __init__(self, dictionary):
            super().__init__()
            self.dictionary = dictionary

    class FairseqCriterion(nn.Module):
        def __init__(self, task):
            super().__init__()
            self.task = task

    class FairseqOptimizer(object):
        def __init__(self, cfg):
            self.cfg = cfg

    class FairseqDataclass(object):
        pass

    class _Metrics:
        @staticmethod
        def log_scalar(*a, **k):
            pass

        @staticmethod
        def log_derived(*a, **k):
            pass

    metrics = _Metrics()

    def _register(name, dataclass=None):
        def deco(cls):
            cls._registered_name = name
            REGISTRY[name] = cls
            return cls
        return deco

    REGISTRY = {}
    register_model = register_criterion = register_optimizer = _register
