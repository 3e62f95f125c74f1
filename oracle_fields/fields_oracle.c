/* fields_oracle.c -- CPU checker of vgicp_prep_approximate_voxel_grid_fields and vgicp_prep_voxel_grid (include/vgicp_prep_b200.h).
 * TEST INFRASTRUCTURE ONLY, like oracle/vgicp_oracle.c, whose orc_approximate_voxel_grid it extends (that function stays as it is).
 *
 * pcl::ApproximateVoxelGrid<PointT> with setDownsampleAllData(true) (PCL's default) averages every field of the point over the voxel,
 * not only x y z.  PCL is not vendored: restated from the published algorithm (pcl/filters/impl/approximate_voxel_grid.hpp) as
 * orc_approximate_voxel_grid restates it, with F float fields summed in float in input order next to x y z and divided once by
 * (float)count at the same flushes.  PCL itself is not on disk, so per-field parity with PCL is not pinned: only the x y z bytes
 * are (they must equal orc_approximate_voxel_grid's, which reproduces the reference's point counts).
 * Compiled without contraction and without fast math, as the oracle is. */
#include <stdlib.h>
#include <math.h>

#if defined(_WIN32)
#define ORC_API
#else
#define ORC_API __attribute__((visibility("default")))
#endif

#define ORC_MAX_FIELDS 8

/* rec: n records of stride_f floats, x y z in floats 0, 1, 2 and field j in float cols[j] (n_fields 0 ... 8).
 * remove_near_origin != 0 first drops the points with (x*x + y*y) + z*z < 1e-3 (src/align.cpp:128-133; stable, so it is the
 * same as filtering first).  out: capacity n records of 3 + n_fields floats, x y z f_0 ... f_{F-1}.
 * Returns the number of output records, or -1 for a bad argument. */
ORC_API int orc_approximate_voxel_grid_fields(const float* rec, int n, int stride_f, const int* cols, int n_fields, float leaf, int histsize, int remove_near_origin,
                                              float* out) {
  typedef struct { int ix, iy, iz, count; float sx, sy, sz; float sf[ORC_MAX_FIELDS]; } He;
  if (n_fields < 0 || n_fields > ORC_MAX_FIELDS || stride_f < 3) return -1;
  for (int j = 0; j < n_fields; j++)
    if (cols[j] < 3 || cols[j] >= stride_f) return -1;
  He* hist = (He*)calloc((size_t)histsize, sizeof(He));
  const int F = n_fields, R = 3 + n_fields;
  const float inv = 1.0f / leaf;
  int m = 0;
  for (int i = 0; i < n; i++) {
    const float* p = rec + (size_t)i * stride_f;
    const float x = p[0], y = p[1], z = p[2];
    if (remove_near_origin && (x * x + y * y) + z * z < 1e-3f) continue;
    const int ix = (int)floorf(x * inv), iy = (int)floorf(y * inv), iz = (int)floorf(z * inv);
    const long long hl = (long long)ix * 7171 + (long long)iy * 3079 + (long long)iz * 4231;
    He* h = &hist[(size_t)(hl & (long long)(histsize - 1))];
    if (h->count && (h->ix != ix || h->iy != iy || h->iz != iz)) {
      const float c = (float)h->count;
      float* o = out + (size_t)m * R;
      o[0] = h->sx / c; o[1] = h->sy / c; o[2] = h->sz / c;
      for (int j = 0; j < F; j++) o[3 + j] = h->sf[j] / c;
      m++;
      h->count = 0; h->sx = h->sy = h->sz = 0.0f;
      for (int j = 0; j < F; j++) h->sf[j] = 0.0f;
    }
    h->ix = ix; h->iy = iy; h->iz = iz;
    h->count++;
    h->sx += x; h->sy += y; h->sz += z;
    for (int j = 0; j < F; j++) h->sf[j] += p[cols[j]];
  }
  for (int s = 0; s < histsize; s++) {
    He* h = &hist[s];
    if (!h->count) continue;
    const float c = (float)h->count;
    float* o = out + (size_t)m * R;
    o[0] = h->sx / c; o[1] = h->sy / c; o[2] = h->sz / c;
    for (int j = 0; j < F; j++) o[3 + j] = h->sf[j] / c;
    m++;
  }
  free(hist);
  return m;
}

/* pcl::VoxelGrid<PointT> (the exact grid) with per-point float fields: the checker of vgicp_prep_voxel_grid, written as the plain
 * serial algorithm of the recipe in include/vgicp_prep_b200.h -- keep, cells, box, index, stable sort, sums.
 * rec, stride_f, cols, n_fields, remove_near_origin: as above.  min_points: voxels with fewer points are dropped (0 and 1 keep all).
 * out: capacity n records of 3 + n_fields floats, in ascending voxel index.
 * Returns the number of output records, -1 for a bad argument, -2 for a refused cloud (a kept cell outside the int range, or more
 * than INT32_MAX cells in the box). */
typedef struct { long long idx; int i; } OrcKeyed;

static int orc_keyed_cmp(const void* a, const void* b) {
  const OrcKeyed* p = (const OrcKeyed*)a;
  const OrcKeyed* q = (const OrcKeyed*)b;
  if (p->idx != q->idx) return p->idx < q->idx ? -1 : 1;
  return p->i < q->i ? -1 : (p->i > q->i);  /* ties in input order: a stable sort */
}

ORC_API int orc_voxel_grid_fields(const float* rec, int n, int stride_f, const int* cols, int n_fields, float leaf, int remove_near_origin, unsigned min_points,
                                  float* out) {
  if (n < 0 || n_fields < 0 || n_fields > ORC_MAX_FIELDS || stride_f < 3 || !(leaf > 0.0f) || !isfinite(leaf)) return -1;
  for (int j = 0; j < n_fields; j++)
    if (cols[j] < 3 || cols[j] >= stride_f) return -1;
  const int R = 3 + n_fields;
  const float inv = 1.0f / leaf;
  int* cell = (int*)malloc(sizeof(int) * 3 * (size_t)(n > 0 ? n : 1));
  OrcKeyed* key = (OrcKeyed*)malloc(sizeof(OrcKeyed) * (size_t)(n > 0 ? n : 1));
  int kept = 0, lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0}, m = 0;
  /* 1-2. kept points and their cells */
  for (int i = 0; i < n; i++) {
    const float* p = rec + (size_t)i * stride_f;
    const float x = p[0], y = p[1], z = p[2];
    if (!isfinite(x) || !isfinite(y) || !isfinite(z)) continue;
    if (remove_near_origin && (x * x + y * y) + z * z < 1e-3f) continue;
    const float v[3] = {x, y, z};
    for (int a = 0; a < 3; a++) {
      const float c = floorf(v[a] * inv);
      if (!(c >= -2147483648.0f && c < 2147483648.0f)) {
        m = -2;
        goto done;
      }
      cell[3 * kept + a] = (int)c;
    }
    key[kept].i = i;
    kept++;
  }
  if (kept == 0) goto done;
  /* 3. box */
  for (int a = 0; a < 3; a++) lo[a] = hi[a] = cell[a];
  for (int k = 1; k < kept; k++)
    for (int a = 0; a < 3; a++) {
      if (cell[3 * k + a] < lo[a]) lo[a] = cell[3 * k + a];
      if (cell[3 * k + a] > hi[a]) hi[a] = cell[3 * k + a];
    }
  {
    const long long dx = (long long)hi[0] - lo[0] + 1, dy = (long long)hi[1] - lo[1] + 1, dz = (long long)hi[2] - lo[2] + 1;
    if (dx > 0x7fffffffLL || dy > 0x7fffffffLL / dx || dz > 0x7fffffffLL / (dx * dy)) {
      m = -2;
      goto done;
    }
    /* 4. voxel index */
    for (int k = 0; k < kept; k++)
      key[k].idx = ((long long)cell[3 * k] - lo[0]) + ((long long)cell[3 * k + 1] - lo[1]) * dx + ((long long)cell[3 * k + 2] - lo[2]) * dx * dy;
  }
  /* 5. stable sort by index, runs of equal index */
  qsort(key, (size_t)kept, sizeof(OrcKeyed), orc_keyed_cmp);
  for (int s = 0; s < kept;) {
    int e = s + 1;
    while (e < kept && key[e].idx == key[s].idx) e++;
    if ((unsigned)(e - s) >= min_points) {
      /* 6. centroids: sums in float in input order, one division by (float)count */
      float* o = out + (size_t)m * R;
      for (int c = 0; c < R; c++) {
        const int col = c < 3 ? c : cols[c - 3];
        float acc = 0.0f;
        for (int k = s; k < e; k++) acc += rec[(size_t)key[k].i * stride_f + col];
        o[c] = acc / (float)(e - s);
      }
      m++;
    }
    s = e;
  }
done:
  free(cell);
  free(key);
  return m;
}
