"""tecogan_b200 -- H100-native (sm_90a) implementation of TecoGAN's recurrent video-SR hot path.

Layout: csrc/ (CUDA kernels + C ABI -> libteco.so), _ffi.py (ctypes binding), variables.py (TF-style
variable scopes holding the weights), lib/{ops,frvsr,Teco,dataloader}.py (host-side mirror of the reference's
Python interface), engine.py (streaming inference recurrence on CUDA graphs), train.py (training step + DP).
There is no CPU fallback anywhere in this package.
"""
__version__ = "0.1.0"
