// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).
// Line-by-line restatement of the Velodyne branch of Laser_feature::laserCloudHandler (loam_livox/source/laser_feature_extractor.hpp:393-825,
// lidar_type != "livox"), with the literal reset-order curvature loop (:524-598) and the insertion sort (:643-654).  The stated deviations
// of the device path are applied here too: the result is defined on the kept points (cloudSize after the filter), the neighbour walks stop at
// the ends of the cloud, fewer than 5 kept points skip the curvature loop, and a coordinate of magnitude above 1e36 is removed with the
// non-finite points.  atan / atan2 are pinned to the correctly rounded float of the double function (DESIGN.md §5 (vi), (xv)).
#pragma once
#include <cmath>
#include <vector>
#include "orc_cloud.hpp"

namespace orc {

struct SpinPt { float x, y, z, intensity; };

struct SpinExtractor {
  int scan_line = 16;
  float minimum_range = 0.1f;
  float plane_resolution = 0.4f;
  std::vector<SpinPt> cloud, sharp, less_sharp, flat, less_flat;
  std::vector<int> ring;                   // per point of `cloud`
  std::vector<float> curvature;            // m_pc_curvature (0 outside [5, N-5))
  std::vector<int> picked_before;          // m_pc_neighbor_picked after :598 (0 outside [5, N-5))
  std::vector<int> label;                  // m_pc_cloud_label after the selection (0 outside [5, N-5))

  static float ori_of(float x, float y) { return -(float)std::atan2((double)y, (double)x); }

  void extract(const float* raw4, int n) {
    const double PI = 3.14159265358979323846;
    // :399-400
    std::vector<SpinPt> in;
    for (int i = 0; i < n; i++) {
      const float* p = raw4 + (size_t)i * 4;
      if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) continue;
      if (std::fabs(p[0]) > 1e36f || std::fabs(p[1]) > 1e36f || std::fabs(p[2]) > 1e36f) continue;
      const float thres = minimum_range;
      if (p[0] * p[0] + p[1] * p[1] + p[2] * p[2] < thres * thres) continue;
      in.push_back({p[0], p[1], p[2], p[3]});
    }
    size_t cloudSize = in.size();
    std::vector<std::vector<SpinPt>> scans(scan_line);
    if (cloudSize > 0) {
      float startOri = ori_of(in[0].x, in[0].y);
      float endOri = (float)((double)ori_of(in[cloudSize - 1].x, in[cloudSize - 1].y) + 2 * PI);
      if (endOri - startOri > 3 * PI) endOri = (float)(endOri - 2 * PI);
      else if (endOri - startOri < PI) endOri = (float)(endOri + 2 * PI);
      bool halfPassed = false;
      for (size_t i = 0; i < cloudSize; i++) {
        SpinPt point = in[i];
        float angle = (float)((double)((float)std::atan((double)(point.z / std::sqrt(point.x * point.x + point.y * point.y))) * 180) / PI);
        int scanID = 0;
        if (scan_line == 16) {
          scanID = int((angle + 15) / 2 + 0.5);
          if (scanID > (scan_line - 1) || scanID < 0) continue;
        } else {
          if (angle >= -8.83) scanID = int((2 - angle) * 3.0 + 0.5);
          else scanID = scan_line / 2 + int((-8.83 - angle) * 2.0 + 0.5);
          if (angle > 2 || angle < -24.33 || scanID > 50 || scanID < 0) continue;
        }
        float ori = ori_of(point.x, point.y);
        if (!halfPassed) {
          if (ori < startOri - PI / 2) ori = (float)(ori + 2 * PI);
          else if (ori > startOri + PI * 3 / 2) ori = (float)(ori - 2 * PI);
          if (ori - startOri > PI) halfPassed = true;
        } else {
          ori = (float)(ori + 2 * PI);
          if (ori < endOri - PI * 3 / 2) ori = (float)(ori + 2 * PI);
          else if (ori > endOri + PI / 2) ori = (float)(ori - 2 * PI);
        }
        float relTime = (ori - startOri) / (endOri - startOri);
        point.intensity = (float)(scanID + 0.1 * relTime);
        scans[scanID].push_back(point);
      }
    }
    // :510-521
    cloud.clear(); ring.clear();
    std::vector<int> scanStartInd(scan_line), scanEndInd(scan_line);
    for (int i = 0; i < scan_line; i++) {
      scanStartInd[i] = (int)cloud.size() + 5;
      for (const SpinPt& p : scans[i]) { cloud.push_back(p); ring.push_back(i); }
      scanEndInd[i] = (int)cloud.size() - 6;
    }
    const int N = (int)cloud.size();
    // :524-598, the literal loop over arrays one longer than the cloud (the forward marks of the last iteration reach index N)
    std::vector<float> curv(N + 7, 0.f);
    std::vector<int> sort_idx(N + 7, 0), picked(N + 7, 0), lab(N + 7, 0);
    const std::vector<SpinPt>& c = cloud;
    for (int i = 5; i < N - 5; i++) {
      float diffX = c[i - 5].x + c[i - 4].x + c[i - 3].x + c[i - 2].x + c[i - 1].x - 10 * c[i].x + c[i + 1].x + c[i + 2].x + c[i + 3].x + c[i + 4].x + c[i + 5].x;
      float diffY = c[i - 5].y + c[i - 4].y + c[i - 3].y + c[i - 2].y + c[i - 1].y - 10 * c[i].y + c[i + 1].y + c[i + 2].y + c[i + 3].y + c[i + 4].y + c[i + 5].y;
      float diffZ = c[i - 5].z + c[i - 4].z + c[i - 3].z + c[i - 2].z + c[i - 1].z - 10 * c[i].z + c[i + 1].z + c[i + 2].z + c[i + 3].z + c[i + 4].z + c[i + 5].z;
      float diff = diffX * diffX + diffY * diffY + diffZ * diffZ;
      curv[i] = diff; sort_idx[i] = i; picked[i] = 0; lab[i] = 0;
      if (diff > 0.1) {
        float depth1 = std::sqrt(c[i].x * c[i].x + c[i].y * c[i].y + c[i].z * c[i].z);
        float depth2 = std::sqrt(c[i + 1].x * c[i + 1].x + c[i + 1].y * c[i + 1].y + c[i + 1].z * c[i + 1].z);
        if (depth1 > depth2) {
          diffX = c[i + 1].x - c[i].x * depth2 / depth1;
          diffY = c[i + 1].y - c[i].y * depth2 / depth1;
          diffZ = c[i + 1].z - c[i].z * depth2 / depth1;
          if (std::sqrt(diffX * diffX + diffY * diffY + diffZ * diffZ) / depth2 < 0.1)
            for (int k = i - 5; k <= i; k++) picked[k] = 1;
        } else {
          diffX = c[i + 1].x * depth1 / depth2 - c[i].x;
          diffY = c[i + 1].y * depth1 / depth2 - c[i].y;
          diffZ = c[i + 1].z * depth1 / depth2 - c[i].z;
          if (std::sqrt(diffX * diffX + diffY * diffY + diffZ * diffZ) / depth1 < 0.1)
            for (int k = i + 1; k <= i + 6; k++) picked[k] = 1;
        }
      }
      float diffX2 = c[i].x - c[i - 1].x, diffY2 = c[i].y - c[i - 1].y, diffZ2 = c[i].z - c[i - 1].z;
      float diff2 = diffX2 * diffX2 + diffY2 * diffY2 + diffZ2 * diffZ2;
      float dis = c[i].x * c[i].x + c[i].y * c[i].y + c[i].z * c[i].z;
      if (diff > 0.0002 * dis && diff2 > 0.0002 * dis) picked[i] = 1;
    }
    curvature.assign(N, 0.f); picked_before.assign(N, 0);
    for (int i = 5; i < N - 5; i++) { curvature[i] = curv[i]; picked_before[i] = picked[i]; }
    // :631-768
    sharp.clear(); less_sharp.clear(); flat.clear(); less_flat.clear();
    const float sharp_point_threshold = 0.05;
    auto gap = [&](int a, int b) { float dx = c[a].x - c[b].x, dy = c[a].y - c[b].y, dz = c[a].z - c[b].z; return dx * dx + dy * dy + dz * dz > 0.05; };
    for (int i = 0; i < scan_line; i++) {
      std::vector<SpinPt> lf_scan;
      for (int j = 0; j < 6; j++) {
        int sp = (scanStartInd[i] * (6 - j) + scanEndInd[i] * j) / 6;
        int ep = (scanStartInd[i] * (5 - j) + scanEndInd[i] * (j + 1)) / 6 - 1;
        for (int k = sp + 1; k <= ep; k++)
          for (int l = k; l >= sp + 1; l--)
            if (curv[sort_idx[l]] < curv[sort_idx[l - 1]]) std::swap(sort_idx[l - 1], sort_idx[l]);
        int largestPickedNum = 0;
        for (int k = ep; k >= sp; k--) {
          int ind = sort_idx[k];
          if (picked[ind] == 0 && curv[ind] > sharp_point_threshold * 10) {
            largestPickedNum++;
            if (largestPickedNum <= 20) { lab[ind] = 2; sharp.push_back(c[ind]); less_sharp.push_back(c[ind]); }
            else if (largestPickedNum <= 200) { lab[ind] = 1; less_sharp.push_back(c[ind]); }
            else break;
            picked[ind] = 1;
            float times = 100;
            for (int l = 1; l <= 5 * times; l++) { if (ind + l > N - 1 || gap(ind + l, ind + l - 1)) break; picked[ind + l] = 1; }
            for (int l = -1; l >= -5 * times; l--) { if (ind + l < 0 || gap(ind + l, ind + l + 1)) break; picked[ind + l] = 1; }
          }
        }
        int smallestPickedNum = 0;
        for (int k = sp; k <= ep; k++) {
          int ind = sort_idx[k];
          if (picked[ind] == 0 && curv[ind] < sharp_point_threshold) {
            lab[ind] = -1; flat.push_back(c[ind]);
            smallestPickedNum++;
            if (smallestPickedNum >= 5) break;
            picked[ind] = 1;
            for (int l = 1; l <= 5; l++) { if (ind + l > N - 1 || gap(ind + l, ind + l - 1)) break; picked[ind + l] = 1; }
            for (int l = -1; l >= -5; l--) { if (ind + l < 0 || gap(ind + l, ind + l + 1)) break; picked[ind + l] = 1; }
          }
        }
        for (int k = sp; k <= ep; k++) if (lab[k] <= 0) lf_scan.push_back(c[k]);
      }
      // :771-776
      std::vector<float> ds(lf_scan.size() * 4);
      const int m = voxel_grid((const float*)lf_scan.data(), (int)lf_scan.size(), plane_resolution / 2, ds.data());
      for (int k = 0; k < m; k++) less_flat.push_back({ds[4 * k], ds[4 * k + 1], ds[4 * k + 2], ds[4 * k + 3]});
    }
    label.assign(N, 0);
    for (int i = 5; i < N - 5; i++) label[i] = lab[i];
  }
};

}  // namespace orc
