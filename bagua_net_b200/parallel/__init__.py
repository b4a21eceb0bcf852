"""Symmetric-memory communicator and the data-parallel engine built on the fused kernels."""
from .comm import SymmComm, init_process_group_from_env  # noqa: F401
from .ddp import BnetDDP, no_weight_decay_groups  # noqa: F401
