// features_harness.cpp -- TEST-ONLY serial build of locus_b200/csrc/features.h with g++: the feature extraction of
// PointCloudFilter::Filter driven one point / one ring at a time through the same scalar functions the kernels of
// features.cu call, so that tests/test_features_cpu.py can check them against the oracle bit for bit without a GPU.
// usage: features_harness in.bin out.bin n_rings lower upper scan_period cr regions max_sharp max_less_sharp max_flat
//        curvature_threshold leaf      (in.bin: n x 3 float32; out.bin: m x 4 float32; stdout: the six counts)
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "features.h"

using namespace lb;

int main(int argc, char** argv) {
  if (argc != 14) { std::fprintf(stderr, "usage: see the header\n"); return 2; }
  FeatParams p;
  p.n_rings = std::atoi(argv[3]); p.lower = std::strtof(argv[4], nullptr); p.upper = std::strtof(argv[5], nullptr);
  p.scan_period = std::strtof(argv[6], nullptr); p.cr = std::atoi(argv[7]); p.n_regions = std::atoi(argv[8]);
  p.max_sharp = std::atoi(argv[9]); p.max_less_sharp = std::atoi(argv[10]); p.max_flat = std::atoi(argv[11]);
  p.curv_thr = std::strtof(argv[12], nullptr); p.leaf = std::strtof(argv[13], nullptr);
  p.factor = (float)(p.n_rings - 1) / (p.upper - p.lower);
  std::vector<float> xyz;
  {
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    float v;
    while (std::fread(&v, sizeof(float), 1, f) == 1) xyz.push_back(v);
    std::fclose(f);
  }
  const size_t n = xyz.size() / 3;
  if (n == 0) return 2;
  float so, eo;
  feat_scan_bounds(xyz[0], xyz[1], xyz[3 * (n - 1)], xyz[3 * (n - 1) + 1], so, eo);
  // halfPassed: the first kept point whose branch-A orientation passes half a turn
  size_t cut = (size_t)-1;
  for (size_t i = 0; i < n && cut == (size_t)-1; i++) {
    float x, y, z;
    if (feat_ring(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], p, x, y, z) >= 0 && feat_half_passes(feat_ori_a(x, z, so), so)) cut = i;
  }
  std::vector<std::vector<f4>> rings(p.n_rings);
  size_t arranged = 0;
  for (size_t i = 0; i < n; i++) {
    float x, y, z;
    const int r = feat_ring(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], p, x, y, z);
    if (r < 0) continue;
    const float ori = i <= cut ? feat_ori_a(x, z, so) : feat_ori_b(x, z, eo);
    rings[r].push_back(f4{x, y, z, feat_intensity(r, ori, so, eo, p.scan_period)});
    arranged++;
  }
  std::vector<f4> cat[4];
  for (int r = 0; r < p.n_rings; r++) {
    const std::vector<f4>& P = rings[r];
    const long long cnt = (long long)P.size();
    if (feat_ring_skipped(cnt, p.cr)) continue;
    std::vector<unsigned char> picked(cnt, 0);
    std::vector<signed char> label(cnt, FEAT_NO_REGION);
    std::vector<float> curv(cnt, 0.f);
    for (long long i = p.cr; i < cnt - 1 - p.cr; i++) feat_unreliable_marks(P.data(), i, p.cr, picked.data());
    for (long long i = p.cr; i <= cnt - 1 - p.cr; i++) curv[i] = feat_curvature(P.data(), i, p.cr);
    for (int j = 0; j < p.n_regions; j++) {
      long long sp, ep;
      feat_region(cnt, p.cr, p.n_regions, j, sp, ep);
      if (ep <= sp) continue;
      std::vector<long long> order(ep - sp + 1);
      for (long long k = sp; k <= ep; k++) { order[feat_region_rank(curv.data(), sp, ep, k)] = k; label[k] = FEAT_SURFACE_LESS_FLAT; }
      int taken = 0;
      for (size_t k = order.size(); k > 0 && taken < p.max_less_sharp;) {
        const long long idx = order[--k];
        if (!feat_corner_candidate(picked[idx], curv[idx], p.curv_thr)) continue;
        taken++;
        if (taken <= p.max_sharp) { label[idx] = FEAT_CORNER_SHARP; cat[0].push_back(P[idx]); }
        else label[idx] = FEAT_CORNER_LESS_SHARP;
        cat[1].push_back(P[idx]);
        feat_mark_as_picked(P.data(), idx, p.cr, picked.data());
      }
      taken = 0;
      for (size_t k = 0; k < order.size() && taken < p.max_flat; k++) {
        const long long idx = order[k];
        if (!feat_flat_candidate(picked[idx], curv[idx], p.curv_thr)) continue;
        taken++;
        label[idx] = FEAT_SURFACE_FLAT;
        cat[2].push_back(P[idx]);
        feat_mark_as_picked(P.data(), idx, p.cr, picked.data());
      }
    }
    std::vector<f4> lf;
    for (long long k = 0; k < cnt; k++) if (label[k] <= FEAT_SURFACE_LESS_FLAT) lf.push_back(P[k]);
    if (lf.empty()) continue;
    float mn[3] = {lf[0].x, lf[0].y, lf[0].z}, mx[3] = {lf[0].x, lf[0].y, lf[0].z};
    for (const f4& q : lf) {
      const float v[3] = {q.x, q.y, q.z};
      for (int d = 0; d < 3; d++) { mn[d] = std::min(mn[d], v[d]); mx[d] = std::max(mx[d], v[d]); }
    }
    const FeatGrid g = feat_grid(mn, mx, p.leaf);
    if (g.overflow) { cat[3].insert(cat[3].end(), lf.begin(), lf.end()); continue; }
    std::vector<std::pair<int, size_t>> kv;
    for (size_t k = 0; k < lf.size(); k++) kv.push_back({feat_voxel_key(g, lf[k].x, lf[k].y, lf[k].z), k});
    std::sort(kv.begin(), kv.end());
    for (size_t s = 0; s < kv.size();) {
      size_t e = s + 1;
      f4 acc = lf[kv[s].second];
      for (; e < kv.size() && kv[e].first == kv[s].first; e++) {
        const f4& q = lf[kv[e].second];
        acc.x = acc.x + q.x; acc.y = acc.y + q.y; acc.z = acc.z + q.z; acc.w = acc.w + q.w;
      }
      const float c = (float)(e - s);
      cat[3].push_back(f4{acc.x / c, acc.y / c, acc.z / c, acc.w / c});
      s = e;
    }
  }
  float T[12];
  feat_rotation(T);
  FILE* f = std::fopen(argv[2], "wb");
  if (!f) return 2;
  size_t total = 0;
  for (int c = 0; c < 4; c++)
    for (const f4& q : cat[c]) {
      float o[4];
      xform_pcl(T, q.x, q.y, q.z, o[0], o[1], o[2]);
      o[3] = q.w;
      std::fwrite(o, sizeof(float), 4, f);
      total++;
    }
  std::fclose(f);
  std::printf("%zu %zu %zu %zu %zu %zu\n", arranged, cat[0].size(), cat[1].size(), cat[2].size(), cat[3].size(), total);
  return 0;
}
