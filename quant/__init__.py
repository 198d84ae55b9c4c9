"""Import-path compatibility with the reference checkout: `from quant.new_pack import ...`, `from quant.matmul import
...` (models/llama_kivi.py:9-10) resolve to the H100-native implementations of kivi_b200 (libkivi_b200.so)."""
