/* The reference's C example (example/cbindings1/main.cc: three rows of three 1-byte scalars committed
 * over the built-in generators), written against include/blitzar_b200.h in plain C99. It also shows the
 * fixed-generator handle API. Build: gcc -std=c99 -Iinclude examples/cbindings1.c -Lblitzar_b200/lib
 * -lblitzar_b200 -o cbindings1   (run on a machine with an H100; the library has no CPU fallback). */
#include <stdio.h>
#include <string.h>

#include "blitzar_b200.h"

int main(void) {
  const struct sxt_config config = {SXT_GPU_BACKEND, 0};
  if (sxt_init(&config) != 0) {
    fprintf(stderr, "sxt_init failed\n");
    return 1;
  }

  /* three commitments: rows of a 3 x 3 table of 1-byte scalars */
  const uint8_t data[3][3] = {{1, 2, 3}, {4, 5, 6}, {7, 8, 9}};
  struct sxt_sequence_descriptor descriptors[3];
  for (int i = 0; i < 3; ++i) {
    descriptors[i].element_nbytes = 1;
    descriptors[i].n = 3;
    descriptors[i].data = data[i];
    descriptors[i].is_signed = 0;
  }
  struct sxt_ristretto255_compressed commitments[3];
  sxt_curve25519_compute_pedersen_commitments(commitments, 3, descriptors, 0);
  for (int i = 0; i < 3; ++i) {
    printf("commitment %d: ", i);
    for (int k = 0; k < 32; ++k)
      printf("%02x", commitments[i].ristretto_bytes[k]);
    printf("\n");
  }

  /* the same first commitment through a fixed-generator handle over g(0), g(1), g(2) */
  struct sxt_ristretto255 generators[3];
  if (sxt_ristretto255_get_generators(generators, 3, 0) != 0)
    return 1;
  struct sxt_multiexp_handle* handle = sxt_multiexp_handle_new(SXT_CURVE_RISTRETTO255, generators, 3);
  struct sxt_ristretto255 result;
  sxt_fixed_multiexponentiation(&result, handle, 1, 1, 3, data[0]);
  sxt_multiexp_handle_free(handle);
  printf("fixed-base result X[0] = %llu\n", (unsigned long long)result.X[0]);
  return 0;
}
