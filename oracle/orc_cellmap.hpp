// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header). PARITY UNPINNED.
// CPU restatement of the voxel-cell map as the matching path uses it (matching_mode 1):
//   loam_livox/source/cell_map_keyframe.hpp
//     :556-571 find_cell_center     (cell centre = round((p - r/4) / (r/2)) * (r/2) + r/4 with r/2 stored by set_resolution :674-679)
//     :619-672 append_cloud, :578-617 set_point_cloud (first call; bumps the frame index twice)
//     :716-758 find_cell (revisit: a cell not touched for >= m_minimum_revisit_threshold frames is replaced by a fresh one)
//     :681-714 add_cell, :378-419 append_pt, :331-351 get_pointcloud / set_pointcloud (cells keep xyz only: intensity becomes 0)
//     :761-788 find_cells_in_radius (PCL octree radius search over the cell centres, squared float distance <= r^2)
//   loam_livox/source/laser_mapping.hpp
//     :310-324 if_pt_in_fov, :471-516 update_buff_for_matching, matching_mode 1 (per-cell VoxelGrid, down-sample-and-replace)
// Deviation (documented): the octree returns cells in an unspecified order; the oracle visits them in ascending (k, j, i) cell-index order.
#pragma once
#include <cmath>
#include <cstdint>
#include <map>
#include <tuple>
#include <vector>
#include "orc_cloud.hpp"
#include "orc_math.hpp"

namespace orc {

struct CellMap {
  typedef std::tuple<int, int, int> Key;   // (k, j, i): z, y, x cell index; ascending order = the oracle's visiting order
  struct Cell { std::vector<float> pts; /* xyz triples */ int create_frame = 0, last_update = 0; float center[3]; };
  float resolution = 0.5f;                 // what set_resolution(1.0) stores
  int revisit_threshold = 2147483647;
  int current_frame_idx = 0;
  bool initialized = false;
  std::map<Key, Cell> cells;

  void set_resolution(float r) { resolution = r * 0.5f; }

  static int cell_index(float p, float box, float half) { return (int)std::round((p - half) / box); }
  Key key_of(const float* p) const {
    const float box = resolution * 1.0f, half = resolution * 0.5f;
    return Key(cell_index(p[2], box, half), cell_index(p[1], box, half), cell_index(p[0], box, half));
  }
  void center_of(const Key& k, float c[3]) const {
    const float box = resolution * 1.0f, half = resolution * 0.5f;
    c[0] = (float)std::get<2>(k) * box + half; c[1] = (float)std::get<1>(k) * box + half; c[2] = (float)std::get<0>(k) * box + half;
  }

  Cell& find_cell(const float* p, bool treat_revisit) {   // if_add = 1
    Key k = key_of(p);
    auto it = cells.find(k);
    if (it == cells.end()) {
      Cell c; c.create_frame = current_frame_idx; c.last_update = current_frame_idx; center_of(k, c.center);
      return cells.emplace(k, c).first->second;
    }
    if (treat_revisit) {
      if (current_frame_idx - it->second.last_update < revisit_threshold) it->second.last_update = current_frame_idx;
      else { Cell c; c.create_frame = current_frame_idx; c.last_update = current_frame_idx; center_of(k, c.center); it->second = c; }
    }
    return it->second;
  }

  // pts: n x 4 (x,y,z,intensity); only xyz is kept (pcl_pts_to_eigen_pts)
  void append_cloud(const float* pts, int n) {
    const bool first = cells.empty();
    for (int i = 0; i < n; i++) {
      const float* p = pts + (size_t)i * 4;
      Cell& c = find_cell(p, true);
      c.pts.push_back(p[0]); c.pts.push_back(p[1]); c.pts.push_back(p[2]);
    }
    if (first) { initialized = true; current_frame_idx++; }   // set_point_cloud bumps the index as well
    current_frame_idx++;
  }

  // laser_mapping.hpp:310-324
  static int if_pt_in_fov(const double c[3], const Qd& q_w_curr, const V3d& t_w_curr, float maximum_in_fov_angle) {
    const double n2 = q_w_curr.w * q_w_curr.w + q_w_curr.x * q_w_curr.x + q_w_curr.y * q_w_curr.y + q_w_curr.z * q_w_curr.z;
    Qd inv{q_w_curr.w / n2, -q_w_curr.x / n2, -q_w_curr.y / n2, -q_w_curr.z / n2};   // Eigen Quaternion::inverse()
    V3d d{c[0] - t_w_curr.x, c[1] - t_w_curr.y, c[2] - t_w_curr.z};
    V3d a = qrot(inv, d);
    if (a.x < 0) return 0;
    const double an = std::sqrt(a.x * a.x + (a.y * a.y + a.z * a.z)), bn = 1.0;
    float angle;
    if (an == 0 || bn == 0) angle = 0.0f; else angle = (float)std::acos(std::fabs(a.x * 1.0 + (a.y * 0.0 + a.z * 0.0)) / (an * bn));
    return (angle * 57.3 < maximum_in_fov_angle) ? 1 : 0;
  }

  // update_buff_for_matching, matching_mode 1, for one map (:475-516): cells within `search_range` of t_w_curr and inside the FOV are
  // down-sampled (per-cell VoxelGrid), optionally replaced by their down-sampled version, and concatenated. out: n x 4, intensity 0.
  int assemble(const Qd& q_w_curr, const V3d& t_w_curr, float search_range, float maximum_in_fov_angle, float leaf, bool down_sample_replace,
               std::vector<float>& out, int* cells_in_fov) {
    out.clear(); int nfov = 0;
    const float sp[3] = {(float)t_w_curr.x, (float)t_w_curr.y, (float)t_w_curr.z};
    const double r2 = (double)search_range * (double)search_range;   // radiusSearch(double radius): radius * radius in double
    std::vector<float> in4, tmp;
    for (auto& kv : cells) {
      Cell& c = kv.second;
      const float dx = c.center[0] - sp[0], dy = c.center[1] - sp[1], dz = c.center[2] - sp[2];
      if (!((double)(dx * dx + (dy * dy + dz * dz)) <= r2)) continue;   // float squaredNorm (Eigen order) vs double radius^2
      const double cd[3] = {c.center[0], c.center[1], c.center[2]};
      if (!if_pt_in_fov(cd, q_w_curr, t_w_curr, maximum_in_fov_angle)) continue;
      nfov++;
      const int m = (int)c.pts.size() / 3;
      in4.assign((size_t)m * 4, 0.f);
      for (int i = 0; i < m; i++) { in4[(size_t)i * 4] = c.pts[(size_t)i * 3]; in4[(size_t)i * 4 + 1] = c.pts[(size_t)i * 3 + 1]; in4[(size_t)i * 4 + 2] = c.pts[(size_t)i * 3 + 2]; }
      tmp.assign((size_t)m * 4 + 4, 0.f);
      const int mo = voxel_grid(in4.data(), m, leaf, tmp.data());
      if (down_sample_replace) { c.pts.resize((size_t)mo * 3); for (int i = 0; i < mo; i++) { c.pts[(size_t)i * 3] = tmp[(size_t)i * 4]; c.pts[(size_t)i * 3 + 1] = tmp[(size_t)i * 4 + 1]; c.pts[(size_t)i * 3 + 2] = tmp[(size_t)i * 4 + 2]; } }
      out.insert(out.end(), tmp.begin(), tmp.begin() + (size_t)mo * 4);
    }
    if (cells_in_fov) *cells_in_fov = nfov;
    return (int)out.size() / 4;
  }

  int total_points() const { size_t n = 0; for (auto& kv : cells) n += kv.second.pts.size() / 3; return (int)n; }
};

}  // namespace orc
