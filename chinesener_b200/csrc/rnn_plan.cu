// ner_rnn_plan: the instantiation of each cluster recurrence (bilstm.cu, bilstm_bwd.cu, bigru.cu, bigru_bwd.cu,
// lattice.cu) for a call's shape and the device's SM count.  Each launcher asks it and dispatches on the answer, so the
// plan a test reads is the kernel that runs.
#include "common.cuh"
#include "rnn_cluster.cuh"

namespace {

int lstm_fwd(int B, int H, int sms, int* R, int* C, int* resident) {
  if (H % 4 != 0) return NER_ERR_UNSUPPORTED;
  *C = rnn::lstm_pick_cluster(H);
  if (*C == 0) return NER_ERR_UNSUPPORTED;
  // W_h in registers: one gate column of H fp32 per thread, 4 H / C <= 256 threads (H = 128: bert_bilstm_crf / bilstm_crf)
  *resident = H == 128 && 4 * (H / *C) <= 256;
  const int r = rnn::rows_per_cluster(B, *C, sms);
  if (*resident) {
    // four stacked PREDICT batches (B = 256): 4 rows per cluster would be 256 CTAs = two waves of the one-CTA-per-SM
    // kernel, so 8 (the R = 4 rule implies this one, so R = 4 never runs register-resident)
    *R = (long)2 * ((B + 3) / 4) * *C > sms ? 8 : r == 2 ? 2 : 1;
  } else {
    *R = r;
  }
  return NER_OK;
}

int lstm_bwd(int B, int H, int sms, int* R, int* C, int* resident) {
  *C = rnn::lstm_pick_cluster_bwd(H);
  if (*C == 0 || H / *C > 256) return NER_ERR_UNSUPPORTED;
  *R = rnn::rows_per_cluster(B, *C, sms) >= 2 && 2 * (H / *C) <= 512 ? 2 : 1;
  *resident = H == 128 && *C == 2;   // 4H / 4 = 128 columns of the recurrent matrix per thread
  return NER_OK;
}

int gru(int B, int H, int sms, int* R, int* C) {
  if (H % 4 != 0) return NER_ERR_UNSUPPORTED;
  *C = rnn::gru_pick_cluster(H);
  if (*C == 0) return NER_ERR_UNSUPPORTED;
  *R = rnn::rows_per_cluster(B, *C, sms);
  return NER_OK;
}

}  // namespace

extern "C" int ner_rnn_plan(int kernel, int B, int H, int Kw, int num_sms, int* rows, int* cluster, int* resident) {
  int R = 0, C = 0, res = 0;
  int status = NER_ERR_INVALID_ARG;
  if (B >= 0 && H >= 1 && num_sms >= 1) {
    switch (kernel) {
      case NER_RNN_LSTM_FWD: status = lstm_fwd(B, H, num_sms, &R, &C, &res); break;
      case NER_RNN_LSTM_BWD: status = lstm_bwd(B, H, num_sms, &R, &C, &res); break;
      case NER_RNN_GRU_FWD:
      case NER_RNN_GRU_BWD: status = gru(B, H, num_sms, &R, &C); break;
      case NER_RNN_LATTICE_FWD:
      case NER_RNN_LATTICE_BWD: status = rnn::lattice_config(B, H, Kw, num_sms, &R, &C); break;
      default: break;
    }
  }
  if (status != NER_OK) R = C = res = 0;
  if (rows) *rows = R;
  if (cluster) *cluster = C;
  if (resident) *resident = res;
  return status;
}
