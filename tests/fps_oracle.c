/* fps_oracle.c -- CPU restatement of sgb_id_lists_fps (include/sgb200.h), step by step as the header states it, for the
 * tests. Compiled with -ffp-contract=off, so every float operation is one IEEE single-precision operation, rounded to
 * nearest. Each list is one literal loop; the caller may run ranges of lists on several threads. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static uint64_t fps_key(float d, long long pos) {
  uint32_t u;
  memcpy(&u, &d, 4);
  const uint64_t hi = isnan(d) ? 0u : (uint64_t)u + 1u;
  return (hi << 32) | (uint64_t)(0xFFFFFFFFu - (uint32_t)pos);
}

/* out int32 [n, K]; xyz float32 rows of stride ld */
void orc_id_lists_fps(const long long *off, const int32_t *ids, int n, int N, const float *xyz, long long ld, int K,
                      int32_t *out) {
  for (int k = 0; k < n; k++) {
    int32_t *row = out + (size_t)k * K;
    const long long start = off[k], len = off[k + 1] - off[k];
    for (int j = 0; j < K; j++) row[j] = -1;
    if (len <= 0 || len > 0x7FFFFFFFll) continue;
    long long m = 0;
    for (long long i = 0; i < len; i++) m += (ids[start + i] >= 0 && ids[start + i] < N);
    if (m == 0) continue;
    long long *pos = (long long *)malloc(m * sizeof(long long));
    float *P = (float *)malloc(m * 3 * sizeof(float)), *d = (float *)malloc(m * sizeof(float));
    m = 0;
    for (long long i = 0; i < len; i++) {
      const int32_t id = ids[start + i];
      if (id < 0 || id >= N) continue;
      pos[m] = i;
      for (int c = 0; c < 3; c++) P[3 * m + c] = xyz[(size_t)id * ld + c];
      d[m] = INFINITY;
      m++;
    }
    long long s = 0; /* index into the valid positions: the smallest valid position */
    row[0] = ids[start + pos[s]];
    for (int j = 1; j < K; j++) {
      const float sx = P[3 * s], sy = P[3 * s + 1], sz = P[3 * s + 2];
      uint64_t best = 0;
      long long arg = -1;
      for (long long i = 0; i < m; i++) {
        const float dx = P[3 * i] - sx, dy = P[3 * i + 1] - sy, dz = P[3 * i + 2] - sz;
        const float t = (dx * dx + dy * dy) + dz * dz;
        d[i] = (isnan(d[i]) || isnan(t)) ? NAN : (t < d[i] ? t : d[i]);
        const uint64_t key = fps_key(d[i], pos[i]);
        if (key > best) {
          best = key;
          arg = i;
        }
      }
      s = arg;
      row[j] = ids[start + pos[s]];
    }
    free(pos);
    free(P);
    free(d);
  }
}
