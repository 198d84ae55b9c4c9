"""kivi_b200 -- H100-native (sm_90a) implementation of KIVI's decode hot path.

Host side mirrors the reference's Python surface (quant/new_pack.py, quant/matmul.py, quant/gemv.py,
the `kivi_gemv` extension module, the attention hook of models/llama_kivi.py); all compute runs in
hand-written CUDA behind the C ABI of include/kivi_b200.h (libkivi_b200.so).  No fallbacks.
"""
__version__ = "0.1.0"
