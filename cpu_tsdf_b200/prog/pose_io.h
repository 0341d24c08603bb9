// pose_io.h — camera poses of the `b200_integrate` program: the file formats and the Affine3d arithmetic of
// src/prog/integrate.cpp:452-483, 570, 638.  Eigen is not a dependency; the evaluation orders below restate
// Eigen's [recalled]: Transform::inverse (Affine) = cofactor inverse of the linear part, t' = -(inv * t);
// Transform * Transform (both Affine) = linear * linear, linear * t_rhs + t_lhs; 3-term sums as a0 + (a1 + a2).
#pragma once
#include "../csrc/host_math.h"

#include <array>
#include <fstream>
#include <string>

namespace b200prog {

using Pose = std::array<double, 16>;      // row-major 4x4

inline Pose pose_identity () { Pose p{}; p[0] = p[5] = p[10] = p[15] = 1.0; return p; }

// integrate.cpp:455-474: twelve floats (ascii .txt or binary .transform), rows 0..2; last row 0 0 0 1
inline bool load_pose (const std::string& path, bool binary, Pose& out)
{
  std::ifstream f (path.c_str (), binary ? std::ios::binary : std::ios::in);
  if (!f) return false;
  out = pose_identity ();
  for (int y = 0; y < 3; y++)
    for (int x = 0; x < 4; x++)
    {
      float v = 0.f;
      if (binary) f.read ((char*) &v, sizeof (float)); else f >> v;
      out[y * 4 + x] = static_cast<double> (v);
    }
  return true;
}

inline Pose pose_inverse (const Pose& p)
{
  double r[12];
  b2host::affine_inverse (p.data (), r);
  Pose o = pose_identity ();
  for (int i = 0; i < 12; ++i) o[i] = r[i];
  return o;
}

inline Pose pose_mul (const Pose& a, const Pose& b)
{
  Pose o = pose_identity ();
  for (int i = 0; i < 3; ++i)
  {
    for (int j = 0; j < 3; ++j)
      o[i * 4 + j] = b2host::sum3<double> (a[i * 4 + 0] * b[0 * 4 + j], a[i * 4 + 1] * b[1 * 4 + j], a[i * 4 + 2] * b[2 * 4 + j]);
    o[i * 4 + 3] = b2host::sum3<double> (a[i * 4 + 0] * b[3], a[i * 4 + 1] * b[7], a[i * 4 + 2] * b[11]) + a[i * 4 + 3];
  }
  return o;
}

} // namespace b200prog
