// Status strings and ABI version of libner_b200.so.
#include "common.cuh"
#include <stdio.h>

extern "C" int ner_abi_version(void) { return 2; }   // 2: ner_bert_attention takes n_rows

#ifndef NER_SOURCE_HASH
#define NER_SOURCE_HASH "unknown"
#endif
// "src=<sha256[:16] of csrc/*.cu, csrc/*.cuh, include/*.h> nvcc=<major.minor> arch=sm_90a": what chinesener_b200/build.py
// computed over the tree this object was compiled from (build provenance: the .so files are shipped prebuilt).
extern "C" const char* ner_build_info(void) {
  static char info[128];
  snprintf(info, sizeof(info), "src=%s nvcc=%d.%d arch=sm_90a", NER_SOURCE_HASH, __CUDACC_VER_MAJOR__, __CUDACC_VER_MINOR__);
  return info;
}

extern "C" const char* ner_strerror(int status) {
  static thread_local char buf[160];
  switch (status) {
    case NER_OK: return "ok";
    case NER_ERR_INVALID_ARG: return "invalid argument (null pointer, bad size, misaligned buffer or bad enum)";
    case NER_ERR_UNSUPPORTED: return "unsupported configuration for the sm_90a kernels (e.g. K > 32 tags)";
    case NER_ERR_WORKSPACE: return "workspace missing or too small";
    case NER_ERR_NO_DRIVER: return "CUDA driver entry point cuTensorMapEncodeTiled unavailable";
    default: break;
  }
  if (status <= NER_ERR_CUDA_BASE) {
    const cudaError_t e = static_cast<cudaError_t>(NER_ERR_CUDA_BASE - status);
    snprintf(buf, sizeof(buf), "CUDA error %d: %s", (int)e, cudaGetErrorString(e));
    return buf;
  }
  snprintf(buf, sizeof(buf), "unknown ner_b200 status %d", status);
  return buf;
}
