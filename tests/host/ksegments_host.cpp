// TEST INFRASTRUCTURE ONLY: compiles centerpose_b200/csrc/ksegments.h (the fixed K segments of batch-invariant plans)
// for the host so that tests/test_batch_invariant_cpu.py can check the rule against its restatement.  Never loaded by
// the product.
#include "../../centerpose_b200/csrc/ksegments.h"

extern "C" {

int ks_fixed(long long tiles1, int slabs) { return cp::fixed_ksegments(tiles1, slabs); }
int ks_sms() { return cp::kInvariantSMs; }

}
