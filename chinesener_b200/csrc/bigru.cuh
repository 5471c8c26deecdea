// Launch geometry shared by the GRU recurrence (bigru.cu) and its back-propagation through time (bigru_bwd.cu).  Both
// keep the same recurrent weights resident (three columns per owned unit, four lanes per unit) and exchange at most
// 3 R H floats per step through double-buffered DSMEM, so one cluster size and one shared-memory size serve both.
#pragma once
#include <stddef.h>

#include "common.cuh"

// float4 weight streams of four lanes per unit: ceil(H/8) for the 2H-wide gate columns, ceil(H/16) for the candidate
static inline size_t ner_bigru_smem_bytes(int H, int C, int R) {
  const int NT = 4 * (H / C), H4 = H / 4;
  return (size_t)((H4 + 1) / 2 + (H4 + 3) / 4) * NT * 16 + (size_t)6 * R * H * 4 + 64;   // + s_len[8] + 4 mbarriers
}

// Smallest power-of-two cluster (<= 8, portable) whose slice fits 200 KB at R = 4 with at most 512 threads; 0 if none.
static inline int ner_bigru_pick_cluster(int H) {
  for (int C = 1; C <= 8; C *= 2) {
    if (H % C != 0) continue;
    if (4 * (H / C) <= 512 && ner_bigru_smem_bytes(H, C, 4) <= 200 * 1024) return C;
  }
  return 0;
}

// Rows per cluster: fill the SMs once when the batch is small, amortise the weight reads when it is large.
static inline int ner_bigru_rows_per_cluster(int B, int C) {
  int R = 1;
  if ((long)2 * B * C > ner_num_sms()) R = 2;
  if ((long)2 * ((B + 1) / 2) * C > 2 * ner_num_sms()) R = 4;
  return R;
}
