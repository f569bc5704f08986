// TEST INFRASTRUCTURE — never linked into the product.
//
// Normalising generator ingestion (msm.cuh ingest_normalized) as serial host loops: commitments of
// the device call (CurveOps::commit_device) and of the offsets call (commit_device_offsets) with the
// normalisation on or off (MsmOptions::normalize_gens, BLITZAR_B200_NORMALIZE_GENS in the product),
// and the ingestion itself, so that the device generators it writes can be inspected. Compiled into
// the emulation library next to emul.cpp (blitzar_b200/build.py build_emul); Python side in
// tests/normalize_emul.py.
#include <vector>

#include "emul_prefix.h"
#include "../../blitzar_b200/csrc/engine_api.cuh"
#include "../../blitzar_b200/csrc/msm.cuh"

using namespace b200;

static const CurveVTable& normalize_vt(unsigned curve_id) {
  switch (curve_id) {
  case 0: return kVTableEd25519;
  case 1: return kVTableBls12381;
  case 2: return kVTableBn254;
  default: return kVTableGrumpkin;
  }
}

static EngineCtx normalize_ctx(unsigned normalize) {
  MsmOptions opt;
  opt.normalize_gens = normalize;
  return EngineCtx{0, opt, nullptr, 0};
}

extern "C" {
// b200_commit_device over host pointers in num_ranges generator ranges
void emul_normalize_commit(unsigned curve_id, void* out_commitments, uint32_t num,
                           const sxt_sequence_descriptor* d, const void* generators,
                           unsigned num_ranges, unsigned normalize) {
  if (num == 0) return;
  normalize_vt(curve_id).commit_device(normalize_ctx(normalize), out_commitments, nullptr, num, d,
                                       generators, 0, num_ranges ? num_ranges : 1, nullptr, nullptr);
}
// b200_commit_device_with_offsets over host pointers (offsets null = all 0)
void emul_normalize_commit_offsets(unsigned curve_id, void* out_commitments, uint32_t num,
                                   const sxt_sequence_descriptor* d, const void* generators,
                                   const uint64_t* offsets, unsigned num_ranges,
                                   unsigned normalize) {
  if (num == 0) return;
  normalize_vt(curve_id).commit_device_offsets(normalize_ctx(normalize), out_commitments, nullptr,
                                               num, d, generators, offsets, false,
                                               num_ranges ? num_ranges : 1, nullptr, nullptr);
}
// n ristretto255 ABI generators -> device generators (Ed25519::Gen, 128 bytes each), normalised
// (normalize != 0) or as IngestBody writes them; returns the Z = 0 flag of the normalisation
unsigned emul_ingest_generators(const void* raw, uint64_t n, void* out_gens, unsigned normalize) {
  if (!normalize) {
    launch(IngestBody<Ed25519, false>{(const unsigned char*)raw, (Ed25519::Gen*)out_gens}, n, 0);
    return 0;
  }
  u32 invalid = 0;
  ingest_normalized(0, (const unsigned char*)raw, (Ed25519::Gen*)out_gens, IngestMap{}, n, &invalid);
  return invalid;
}
}
