#!/bin/bash
# Lists the reference translation units the CPU MSM path needs (SURVEY.md Appendix A).
R=${1:?usage: list_sources.sh <reference checkout>}
find $R/sxt/base/{bit,container,error,num,memory,iterator,type,field,curve,functional,device,macro} \
     $R/sxt/memory $R/sxt/execution/{async,device,schedule,kernel} \
     $R/sxt/{field51,curve21,ristretto,scalar25,field12,curve_g1,field25,curve_bng1,fieldgk,curve_gk} \
     $R/sxt/multiexp/{base,index,pippenger,pippenger_multiprod,bitset_multiprod,curve,pippenger2} \
     $R/sxt/seqcommit/generator $R/sxt/cbindings/backend/computational_backend_utility.cc \
     $R/sxt/proof/transcript \
     $R/sxt/proof/inner_product/{cpu_driver,driver,proof_computation,fold,generator_fold,verification_computation,workspace,proof_descriptor}.cc -name '*.cc' ! -name '*.t.cc' \
  | xargs grep -L '<<<\|__global__\|cub/cub' \
  | grep -v 'stacktrace.cc\|/test_\|gpu\|driver_test\|multiexp/curve/multiexponentiation.cc\|multiexp/curve/multiproduct.cc\|scalar25/operation/inner_product.cc\|log_impl.cc\|/log/setup.cc' \
  | sort
