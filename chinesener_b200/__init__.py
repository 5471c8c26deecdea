"""chinesener_b200 — sm_90a kernels behind the bert_bilstm_crf hot path of DSXiangLi/ChineseNER.

Only the hot path lives here: `csrc/` (CUDA kernels + the C-ABI of libner_b200.so),
`_lib.py` (ctypes binding on raw device pointers), `tools/layer.py` (the reference's
layer-function surface) and `model/<name>.py` (the reference's build_graph plugins).
"""
__version__ = "0.1.0"
