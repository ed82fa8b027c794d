"""opendiloco_b200 - an H100-native (sm_90a) DiLoCo training framework with the capabilities of OpenDiLoCo.

    from opendiloco_b200 import LlamaForCausalLM, LlamaConfig, DiLoCoOptimizer, DiLoCoTrainer
"""
from .models.config import LlamaConfig  # noqa: F401
from .models.llama import LlamaForCausalLM  # noqa: F401
from .optim.fused import FusedAdamW, clip_grad_norm_  # noqa: F401
from .optim.muon import FusedMuon  # noqa: F401
from .parallel.diloco import (AllReduceStrategy, DiLoCoGradAverager, DiLoCoOptimizer, DiLoCoStateAverager,  # noqa: F401
                              DiloCoProgressTracker)
from .parallel.swarm import DHT  # noqa: F401
from .trainer import DiLoCoTrainer, TrainerConfig  # noqa: F401

__version__ = "0.1.0"
