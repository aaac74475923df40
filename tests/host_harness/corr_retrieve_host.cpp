// TEST INFRASTRUCTURE: host twin of corr_retrieve_kernel (boxinstseg_b200/csrc/corr.cu).  It compiles the very header the
// kernel is made of (corr_core.cuh: corr_retrieve_query; a phase is a plain loop on the host) with g++ -ffp-contract=off, so
// that the CPU suite can check the batched retrieval -- its arithmetic, the in-level order dependence and the phase
// structure -- against the oracle's sequential Queues.similar on a box without a GPU.  Never shipped.
#include <vector>

#include "../../boxinstseg_b200/csrc/corr_core.cuh"

// corr_retrieve_kernel: the queries of a level one after the other, each with its own scratch (a CTA's shared memory)
extern "C" int host_corr_retrieve(const float* bank_feat, const float* bank_mask, const float* bank_box, const int32_t* bank_ptr,
                                  const int32_t* bank_exists, const int32_t* first, const float* q_feat, const float* q_feat_first,
                                  const float* q_mask, const float* t_feat, const float* t_mask, const float* box,
                                  const int32_t* label, const int32_t* valid, int32_t* src, int32_t* count, int32_t* kcount,
                                  int32_t* slot, int32_t* exists, int64_t n, int64_t num_class, int64_t L, int64_t C, int64_t h,
                                  int64_t w, int64_t Hm, int64_t Wm, float fg_thr, float bg_thr, float app_thr, float ratio_lo,
                                  float ratio_hi, float min_size, int max_objs, int min_objs) {
  const bxs::CorrBank bank{bank_feat, bank_mask, bank_box, bank_ptr, bank_exists, (int)num_class, (int)L};
  const bxs::CorrLevel lvl{q_feat, q_feat_first, q_mask, t_feat, t_mask, box, label, valid, (int)n};
  const bxs::CorrRetrieveCfg cfg{(int)C, (int)h, (int)w, (int)Hm, (int)Wm, fg_thr, bg_thr, app_thr, ratio_lo, ratio_hi, min_size,
                                 max_objs, min_objs};
  const bxs::CorrRetrieveOut out{src, count, kcount, slot, exists};
  std::vector<float> scratch((bxs::corr_retrieve_scratch((int)L, (int)(h * w)) + 3) / 4);
  for (int64_t i = 0; i < n; ++i) bxs::corr_retrieve_query(bank, lvl, cfg, *first, (int)i, scratch.data(), out);
  return 0;
}
