"""diffdock_b200 - H100-native (sm_90a) implementation of DiffDock's score-model hot path: the
TensorProductConvLayer stack + translation/rotation/torsion heads, iterated by the reverse-diffusion sampler.

Drop-in surface (same names/arguments as the reference):
  diffdock_b200.tensor_layers.TensorProductConvLayer   <- models/tensor_layers.py:234
  diffdock_b200.cg_model.CGModel                       <- models/cg_model.py:19
  diffdock_b200.sampling.sampling                      <- utils/sampling.py:69
The arithmetic runs in hand-written CUDA behind the C ABI declared in include/diffdock_b200.h.
"""
__version__ = "0.1.0"
