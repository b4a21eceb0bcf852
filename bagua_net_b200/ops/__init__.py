"""Hand-written sm_90a ops exposed to Python (thin wrappers over libnccl-net.so):

* ``all_reduce``                         — all-reduce of any CUDA tensor by the cheapest route (barrier-free LL words,
                                           in-place NVLS / P2P on heap tensors, staged otherwise); the one-shot and the
                                           fused all-reduce + SGD + broadcast kernels are methods of ``SymmComm``
* ``pack_cast``                          — multi-tensor pack with dtype cast into a flat buffer
* ``ConvBiasReLU``                       — conv + fused bias/ReLU/max-pool forward and backward passes
* ``p2p``                                — the NVLink transport's copy / reduce / cast executor
* ``tc_linear`` / ``tc_conv``            — wgmma/TMA linear (+bias+ReLU, split-K with in-kernel finish), 3x3 convolution
                                           (implicit GEMM, forward + input gradient) and the fused row-parallel GEMM + all-reduce
                                           (import them as ``bagua_net_b200.ops.tc_linear`` / ``.tc_conv``)
"""
from .collectives import all_reduce, pack_cast  # noqa: F401
from .fused_nn import ConvBiasReLU  # noqa: F401
from .p2p import P2PExecutor  # noqa: F401
