// site_score_fam_d.cu -- instantiations: Binomial(total_count, logits), Binomial(total_count, probs)
#include "site_score.cuh"
namespace b2 {
int dispatch_site_d(int family, int dtype, bool grad, const SiteArgs& a, int kind, cudaStream_t s) {
  switch (family) {
    B2_DISPATCH_CASE(kBinomialLogits)
    B2_DISPATCH_CASE(kBinomialProbs)
  }
  return B2_ERR_BAD_FAMILY;
}
}  // namespace b2
