"""lingvo_b200: a Hopper (H100, sm_90a)-native sequence-model framework.

Capability parity target: tensorflow/lingvo (Params / BaseLayer / NestedMap
API, model_registry, trainer/executor entrypoints, checkpoint layout).
Compute path: PyTorch + hand-written sm_90a CUDA kernels + NCCL/NVLink-4.
"""

__version__ = '0.1.0'
