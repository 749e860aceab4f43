// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header). PARITY UNPINNED.
// CPU restatement of the Livox feature extractor:
//   loam_livox/source/livox_feature_extractor.hpp
//     :722-766 extract_laser_features (driver, timestamp bookkeeping)
//     :458-607 projection_scan_3d_2d  (masks, projection, petal split)
//     :343-358 eval_point, :322-341 add_mask_of_point
//     :361-455 compute_features      (5-pt stencil curvature, view angle, labels)
//     :657-719 split_laser_scan      (petal grouping -> only count + first/last idx used)
//     :219-272 get_features          (ordered compaction)
//   loam_livox/include/tools/tools_eigen_math.hpp:25-46 vector_angle
//   loam_livox/source/laser_feature_extractor.hpp:285-335 piece-wise glue
#pragma once
#include <cmath>
#include <cstdint>
#include <vector>

namespace orc {

enum { e_pt_normal = 0, e_pt_000 = 1, e_pt_too_near = 2, e_pt_reflectivity_low = 4, e_pt_reflectivity_high = 8,
       e_pt_circle_edge = 16, e_pt_nan = 32, e_pt_small_view_angle = 64 };
enum { e_label_invalid = -1, e_label_unlabeled = 0, e_label_corner = 1, e_label_surface = 2, e_label_near_nan = 4,
       e_label_near_zero = 8, e_label_hight_intensity = 16 };

struct PtInfo {  // livox_feature_extractor.hpp:118-133
  int pt_type = e_pt_normal; int pt_label = e_label_unlabeled; int idx = 0;
  float raw_intensity = 0.f, time_stamp = 0.f, polar_angle = 0.f; int polar_direction = 0;
  float polar_dis_sq2 = 0.f, depth_sq2 = 0.f, curvature = 0.f, view_angle = 0.f, sigma = 0.f;
  float pt_2d[2] = {0.f, 0.f};  // reference leaves this uninitialised; we define it as 0
};

struct ExtractCfg {
  float thr_corner_curvature = 0.05f, thr_surface_curvature = 0.01f, minimum_view_angle = 10.f;
  float livox_min_allow_dis = 1.0f, livox_min_sigma = 7e-3f;
  float max_fov = 17.f, time_internal_pts = 1.0e-5f;
};

struct Extractor {
  ExtractCfg cfg;
  double first_receive_time = -1, current_time = 0, last_maximum_time_stamp = 0;  // ref leaves the last one uninitialised
  float max_edge_polar_pos = 0;
  std::vector<PtInfo> info; std::vector<float> raw;  // raw: n x 4 (x,y,z,intensity)
  std::vector<int> split_idx; std::vector<float> scan_id_index;
  // petal groups after split_laser_scan: first / last surviving point index per kept petal
  std::vector<int> scan_first_idx, scan_last_idx;

  void add_mask(int idx, int type, int neighbor_count = 0) {  // :322-341
    info[idx].pt_type |= type;
    if (neighbor_count > 0)
      for (int i = -neighbor_count; i < neighbor_count; i++) {
        int j = idx + i;
        if (i != 0 && j >= 0 && j < (int)info.size()) info[j].pt_type |= type;
      }
  }
  void eval_point(int idx) {  // :343-358
    PtInfo& p = info[idx];
    if (p.depth_sq2 < cfg.livox_min_allow_dis * cfg.livox_min_allow_dis) add_mask(idx, e_pt_too_near);
    p.sigma = p.raw_intensity / p.polar_dis_sq2;
    if (p.sigma < cfg.livox_min_sigma) add_mask(idx, e_pt_reflectivity_low);
  }

  int projection_scan_3d_2d(const float* in, int n) {  // :458-607
    info.assign(n, PtInfo()); raw.assign(in, in + (size_t)n * 4);
    scan_id_index.assign(n, 0.f); split_idx.clear();
    std::vector<int> edge_idx, zero_idx;
    for (int idx = 0; idx < n; idx++) {
      const float x = in[idx * 4 + 0], y = in[idx * 4 + 1], z = in[idx * 4 + 2];
      PtInfo* p = &info[idx];
      p->raw_intensity = in[idx * 4 + 3];
      p->idx = idx;
      p->time_stamp = (float)(current_time + (double)(((float)idx) * cfg.time_internal_pts));
      last_maximum_time_stamp = p->time_stamp;
      if (!std::isfinite(x) || !std::isfinite(y) || !std::isfinite(z)) { add_mask(idx, e_pt_nan); continue; }
      if (x == 0) {
        if (idx == 0) { p->pt_2d[0] = 0.01f; p->pt_2d[1] = 0.01f; p->polar_dis_sq2 = 0.0001f; add_mask(idx, e_pt_000); }
        else { p->pt_2d[0] = info[idx - 1].pt_2d[0]; p->pt_2d[1] = info[idx - 1].pt_2d[1]; p->polar_dis_sq2 = info[idx - 1].polar_dis_sq2; add_mask(idx, e_pt_000); continue; }
      }
      p->depth_sq2 = x * x + y * y + z * z;
      p->pt_2d[0] = y / x; p->pt_2d[1] = z / x;
      p->polar_dis_sq2 = p->pt_2d[0] * p->pt_2d[0] + p->pt_2d[1] * p->pt_2d[1];
      eval_point(idx);
      if (p->polar_dis_sq2 > max_edge_polar_pos) add_mask(idx, e_pt_circle_edge, 2);
      if (idx >= 1) {
        float dis_incre = p->polar_dis_sq2 - info[idx - 1].polar_dis_sq2;
        if (dis_incre > 0) p->polar_direction = 1;
        if (dis_incre < 0) p->polar_direction = -1;
        if (p->polar_direction == -1 && info[idx - 1].polar_direction == 1) {
          if (edge_idx.size() == 0 || (idx - split_idx[split_idx.size() - 1]) > 50) { split_idx.push_back(idx); edge_idx.push_back(idx); continue; }
        }
        if (p->polar_direction == 1 && info[idx - 1].polar_direction == -1) {
          if (zero_idx.size() == 0 || (idx - split_idx[split_idx.size() - 1]) > 50) { split_idx.push_back(idx); zero_idx.push_back(idx); continue; }
        }
      }
    }
    split_idx.push_back(n - 1);
    int val_index = 0, pt_angle_index = 0, internal_size = 0; float scan_angle = 0;
    if (split_idx.size() < 6) return 0;
    for (int idx = 0; idx < n; idx++) {
      if ((size_t)val_index < split_idx.size() - 2) {
        if (idx == 0 || idx > split_idx[val_index + 1]) {
          if (idx > split_idx[val_index + 1]) val_index++;
          internal_size = split_idx[val_index + 1] - split_idx[val_index];
          if (info[split_idx[val_index + 1]].polar_dis_sq2 > 10000) pt_angle_index = split_idx[val_index + 1] - (int)(internal_size * 0.20);
          else pt_angle_index = split_idx[val_index + 1] - (int)(internal_size * 0.80);
          scan_angle = (float)(std::atan2(info[pt_angle_index].pt_2d[1], info[pt_angle_index].pt_2d[0]) * 57.3);
          scan_angle = (float)(scan_angle + 180.0);
        }
      }
      info[idx].polar_angle = scan_angle; scan_id_index[idx] = scan_angle;
    }
    return (int)split_idx.size() - 1;
  }

  static float vector_angle_sharp(const float a[3], const float b[3]) {  // tools_eigen_math.hpp:25-46 (force sharp)
    // Eigen's unrolled reduction of a 3-vector (redux_novec_unroller) associates as x + (y + z)
    float an = std::sqrt(a[0] * a[0] + (a[1] * a[1] + a[2] * a[2]));
    float bn = std::sqrt(b[0] * b[0] + (b[1] * b[1] + b[2] * b[2]));
    if (an == 0 || bn == 0) return 0.0f;
    float d = a[0] * b[0] + (a[1] * b[1] + a[2] * b[2]);
    // reference: acosf() of libm (version-dependent last ulp). The oracle pins it to the correctly
    // rounded value, (float)acos((double)c), which is what the CUDA path evaluates as well.
    return (float)std::acos((double)(std::fabs(d) / (an * bn)));
  }

  void compute_features() {  // :361-455
    const size_t n = raw.size() / 4; const size_t ssd = 2; const int critical = e_pt_000 | e_pt_nan;
    if (n < 2 * ssd + 1) return;  // reference underflows size_t here; a scan that small is dropped upstream anyway
    float acc[3];
    for (size_t idx = ssd; idx < n - ssd; idx++) {
      if (info[idx].pt_type & critical) continue;
      acc[0] = acc[1] = acc[2] = 0.f;
      for (size_t i = 1; i <= ssd; i++) {
        if ((info[idx + i].pt_type & e_pt_000) || (info[idx - i].pt_type & e_pt_000)) {
          if (i == 1) info[idx].pt_label |= e_label_near_zero; else info[idx].pt_label = e_label_invalid;
          break;
        } else if ((info[idx + i].pt_type & e_pt_nan) || (info[idx - i].pt_type & e_pt_nan)) {
          if (i == 1) info[idx].pt_label |= e_label_near_nan; else info[idx].pt_label = e_label_invalid;
          break;
        } else {
          acc[0] += raw[(idx + i) * 4 + 0] + raw[(idx - i) * 4 + 0];
          acc[1] += raw[(idx + i) * 4 + 1] + raw[(idx - i) * 4 + 1];
          acc[2] += raw[(idx + i) * 4 + 2] + raw[(idx - i) * 4 + 2];
        }
      }
      if (info[idx].pt_label == e_label_invalid) continue;
      acc[0] -= (float)(ssd * 2) * raw[idx * 4 + 0];
      acc[1] -= (float)(ssd * 2) * raw[idx * 4 + 1];
      acc[2] -= (float)(ssd * 2) * raw[idx * 4 + 2];
      info[idx].curvature = acc[0] * acc[0] + acc[1] * acc[1] + acc[2] * acc[2];
      float va[3] = {raw[idx * 4 + 0], raw[idx * 4 + 1], raw[idx * 4 + 2]};
      float vb[3] = {raw[(idx + ssd) * 4 + 0] - raw[(idx - ssd) * 4 + 0], raw[(idx + ssd) * 4 + 1] - raw[(idx - ssd) * 4 + 1],
                     raw[(idx + ssd) * 4 + 2] - raw[(idx - ssd) * 4 + 2]};
      info[idx].view_angle = (float)(vector_angle_sharp(va, vb) * 57.3);
      if (info[idx].view_angle > cfg.minimum_view_angle) {
        if (info[idx].curvature < cfg.thr_surface_curvature) info[idx].pt_label |= e_label_surface;
        float sq2_diff = 0.1f;
        if (info[idx].curvature > cfg.thr_corner_curvature) {
          if (info[idx].depth_sq2 <= info[idx - ssd].depth_sq2 && info[idx].depth_sq2 <= info[idx + ssd].depth_sq2) {
            if (std::fabs(info[idx].depth_sq2 - info[idx - ssd].depth_sq2) < sq2_diff * info[idx].depth_sq2 ||
                std::fabs(info[idx].depth_sq2 - info[idx + ssd].depth_sq2) < sq2_diff * info[idx].depth_sq2)
              info[idx].pt_label |= e_label_corner;
          }
        }
      }
    }
  }

  // :657-719, reduced to what the caller consumes (petal count, first/last surviving point index per petal).
  void split_laser_scan(int clutter_size) {
    const int n = (int)info.size();
    std::vector<std::vector<int>> scans(clutter_size);
    int scan_idx = 0;
    for (int i = 0; i < n; i++) {
      if (i > 0 && scan_id_index[i] != scan_id_index[i - 1]) scan_idx++;
      if (scan_idx < clutter_size) scans[scan_idx].push_back(i);
    }
    scans.resize(scan_idx);  // reference drops the last petal (laserCloudScans.resize(scan_idx))
    const int remove_type = e_pt_000 | e_pt_too_near | e_pt_nan;
    scan_first_idx.clear(); scan_last_idx.clear();
    for (auto& s : scans) {
      int first = -1, last = -1;
      for (int i : s) if ((info[i].pt_type & remove_type) == 0 && raw[(size_t)i * 4] != 0) { if (first < 0) first = i; last = i; }
      if (first >= 0) { scan_first_idx.push_back(first); scan_last_idx.push_back(last); }
    }
  }

  // :722-766 ; returns number of petal scans handed back to the caller.
  int extract(const float* in, int n, double time_stamp) {
    if (time_stamp <= 0.0000001 || (time_stamp < last_maximum_time_stamp)) current_time = last_maximum_time_stamp;
    else current_time = time_stamp - first_receive_time;
    if (first_receive_time <= 0) first_receive_time = time_stamp;
    max_edge_polar_pos = (float)std::pow(std::tan(cfg.max_fov / 57.3) * 1, 2);
    scan_first_idx.clear(); scan_last_idx.clear();
    int clutter = projection_scan_3d_2d(in, n);
    compute_features();
    if (clutter == 0) return 0;
    split_laser_scan(clutter);
    return (int)scan_first_idx.size();
  }

  // :219-272. Outputs n x 4 float arrays (caller allocates n each).
  void get_features(float minimum_blur, float maximum_blur, float* corners, int* nc, float* surface, int* ns, float* full, int* nf) const {
    const size_t n = info.size();
    int c = 0, s = 0, f = 0;
    float maximum_idx = maximum_blur * n, minimum_idx = minimum_blur * n;
    const int critical = e_pt_000 | e_pt_nan | e_pt_too_near;
    for (size_t i = 0; i < n; i++) {
      if (info[i].idx > maximum_idx || info[i].idx < minimum_idx) continue;
      if ((info[i].pt_type & critical) == 0) {
        if (info[i].pt_label & e_label_corner) {
          if (info[i].pt_type != e_pt_normal) continue;
          if (info[i].depth_sq2 < std::pow(30, 2)) { for (int k = 0; k < 3; k++) corners[c * 4 + k] = raw[i * 4 + k]; corners[c * 4 + 3] = info[i].time_stamp; c++; }
        }
        if (info[i].pt_label & e_label_surface) {
          if (info[i].depth_sq2 < std::pow(1000, 2)) { for (int k = 0; k < 3; k++) surface[s * 4 + k] = raw[i * 4 + k]; surface[s * 4 + 3] = info[i].time_stamp; s++; }
        }
      }
      for (int k = 0; k < 3; k++) full[f * 4 + k] = raw[i * 4 + k];
      full[f * 4 + 3] = info[i].time_stamp; f++;
    }
    *nc = c; *ns = s; *nf = f;
  }

  // laser_feature_extractor.hpp:313-323 — fractional [start,end] of each piece.
  void piece_bounds(int piece_wise, float* start, float* end) const {
    const int nscan = (int)scan_first_idx.size();
    for (int i = 0; i < piece_wise; i++) {
      int start_scans = int((nscan * (i)) / piece_wise);
      int end_scans = int((nscan * (i + 1)) / piece_wise) - 1;
      start[i] = ((float)scan_first_idx[start_scans]) / info.size();
      end[i] = ((float)scan_last_idx[end_scans]) / info.size();
    }
  }
};

}  // namespace orc
