"""disvae on H100: the reference's package surface (disvae/__init__.py:1-3) backed by
hand-written sm_90a kernels (libdisvae_b200.so, C ABI in include/disvae_b200.h)."""
from disvae.models.vae import init_specific_model
from disvae.training import Trainer
from disvae.evaluate import Evaluator

__all__ = ["init_specific_model", "Trainer", "Evaluator"]
