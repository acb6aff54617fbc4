// Host-side true-trajectory generator -- pathgen.path_gen + calc_true_sensor_output +
// parse_motion_def (gnss_ins_sim/pathgen/pathgen.py:26-439), plain C++ on the CPU.
//
// By the north star this stays on the CPU: it is serial in time (a PD attitude controller and
// a low-pass filter on the commands, closed around the integrated state), it runs once per
// experiment and its result is shared by every Monte-Carlo run.  The reference spends ~40 us
// per sample in Python on it (8.6 s for BASELINE config 3, ~10 min for config 4); this
// restatement takes ~0.1 us per sample and removes the last runtime dependency on the
// reference package.  The geomagnetic field itself (WMM at the initial position) is an input:
// gnss_ins_sim_b200/geomag.py evaluates it once on the host.
#pragma once
#include <cmath>
#include <cstdint>

namespace b2ins_host {

constexpr double kRe = 6378137.0;
constexpr double kFlat = 1.0 / 298.257223563;
constexpr double kEcc = 0.0818191908426215;
constexpr double kESqr = kEcc * kEcc;
constexpr double kWie = 7292115e-11;
constexpr double kPi = 3.14159265358979323846;

struct Geo {
  double rm, rn, g, sl, cl;
};
// geoparams.geo_param, geoparams.py:25-53
inline Geo geo_param(double lat, double h) {
  Geo p;
  p.sl = std::sin(lat);
  p.cl = std::cos(lat);
  const double s2 = p.sl * p.sl;
  p.rm = (kRe * (1 - kESqr)) / (std::sqrt(1.0 - kESqr * s2) * (1.0 - kESqr * s2));
  p.rn = kRe / (std::sqrt(1.0 - kESqr * s2));
  const double g1 = 9.7803253359 * (1 + 0.00193185265241 * s2) / std::sqrt(1.0 - kESqr * s2);
  p.g = g1 * (1.0 - (2.0 / kRe) * (1.0 + kFlat + 0.00344978650684 - 2.0 * kFlat * s2) * h +
              3.0 * h * h / kRe / kRe);
  return p;
}
// geoparams.lla2ecef, geoparams.py:70-87
inline void lla2ecef(const double* lla, double* xyz) {
  const double sl = std::sin(lla[0]), cl = std::cos(lla[0]);
  const double r = kRe / std::sqrt(1.0 - kESqr * sl * sl);
  const double rho = (r + lla[2]) * cl;
  xyz[0] = rho * std::cos(lla[1]);
  xyz[1] = rho * std::sin(lla[1]);
  xyz[2] = (r * (1.0 - kESqr) + lla[2]) * sl;
}
// attitude.euler2dcm 'zyx' transposed: b -> n
inline void dcm_b2n(const double* a, double c[3][3]) {
  const double c0 = std::cos(a[0]), c1 = std::cos(a[1]), c2 = std::cos(a[2]);
  const double s0 = std::sin(a[0]), s1 = std::sin(a[1]), s2 = std::sin(a[2]);
  // n->b rows, stored transposed
  c[0][0] = c1 * c0;
  c[1][0] = c1 * s0;
  c[2][0] = -s1;
  c[0][1] = s2 * s1 * c0 - c2 * s0;
  c[1][1] = s2 * s1 * s0 + c2 * c0;
  c[2][1] = c1 * s2;
  c[0][2] = s1 * c2 * c0 + s0 * s2;
  c[1][2] = s1 * c2 * s0 - c0 * s2;
  c[2][2] = c1 * c2;
}
inline void mat_vec(const double c[3][3], const double* v, double* o) {
  for (int i = 0; i < 3; ++i) o[i] = c[i][0] * v[0] + c[i][1] * v[1] + c[i][2] * v[2];
}
inline void mat_t_vec(const double c[3][3], const double* v, double* o) {
  for (int i = 0; i < 3; ++i) o[i] = c[0][i] * v[0] + c[1][i] * v[1] + c[2][i] * v[2];
}
inline void cross(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}
// python float %: result takes the sign of the divisor
inline double py_mod(double x, double m) {
  double r = std::fmod(x, m);
  if (r != 0.0 && ((r < 0.0) != (m < 0.0))) r += m;
  return r;
}
inline double angle_range_pi(double x) {   // attitude.py:799-812
  x = py_mod(x, 2.0 * kPi);
  if (x > kPi) x -= 2.0 * kPi;
  return x;
}
// attitude.euler_angle_range_three_axis, attitude.py:772-797
inline void euler_range(const double* a, double* o) {
  double a1 = a[0], a2 = angle_range_pi(a[1]), a3 = a[2];
  if (a2 > 0.5 * kPi) {
    a2 = kPi - a2;
    a1 += kPi;
    a3 += kPi;
  } else if (a2 < -0.5 * kPi) {
    a2 = -kPi - a2;
    a1 += kPi;
    a3 += kPi;
  }
  o[0] = angle_range_pi(a1);
  o[1] = a2;
  o[2] = angle_range_pi(a3);
}

// calc_true_sensor_output, pathgen.py:331-411
inline void true_sensor_output(const double* pos, const double* vel_b, const double* att,
                               const double c_nb[3][3], const double* vel_dot_b,
                               const double* att_dot, int ref_frame, double g0, double* acc,
                               double* gyro, double* pos_dot) {
  double vel_n[3];
  mat_vec(c_nb, vel_b, vel_n);
  double w_en[3] = {0, 0, 0}, w_ie[3] = {0, 0, 0}, gravity[3] = {0, 0, g0};
  double rm_e = 0, rn_e = 0, cl = 1;
  if (ref_frame == 0) {
    const Geo p = geo_param(pos[0], pos[2]);
    rm_e = p.rm + pos[2];
    rn_e = p.rn + pos[2];
    cl = p.cl;
    gravity[2] = p.g;
    w_en[0] = vel_n[1] / rn_e;
    w_en[1] = -vel_n[0] / rm_e;
    w_en[2] = -vel_n[1] * p.sl / p.cl / rn_e;
    w_ie[0] = kWie * p.cl;
    w_ie[2] = -kWie * p.sl;
  }
  const double sh = std::sin(att[0]), ch = std::cos(att[0]);
  double w_nb[3];
  w_nb[0] = -sh * att_dot[1] + c_nb[0][0] * att_dot[2];
  w_nb[1] = ch * att_dot[1] + c_nb[1][0] * att_dot[2];
  w_nb[2] = att_dot[0] + c_nb[2][0] * att_dot[2];
  if (ref_frame == 0) {
    pos_dot[0] = vel_n[0] / rm_e;
    pos_dot[1] = vel_n[1] / rn_e / cl;
    pos_dot[2] = -vel_n[2];
  } else {
    pos_dot[0] = vel_n[0];
    pos_dot[1] = vel_n[1];
    pos_dot[2] = vel_n[2];
  }
  double w_sum[3] = {w_nb[0] + w_en[0] + w_ie[0], w_nb[1] + w_en[1] + w_ie[1],
                     w_nb[2] + w_en[2] + w_ie[2]};
  mat_t_vec(c_nb, w_sum, gyro);
  double w_ie_b[3], wv[3], tmp[3], gb[3];
  mat_t_vec(c_nb, w_ie, w_ie_b);
  for (int i = 0; i < 3; ++i) tmp[i] = w_ie_b[i] + gyro[i];
  cross(tmp, vel_b, wv);
  mat_t_vec(c_nb, gravity, gb);
  for (int i = 0; i < 3; ++i) acc[i] = vel_dot_b[i] + wv[i] - gb[i];
}

inline double clampd(double v, double lim) { return v > lim ? lim : (v < -lim ? -lim : v); }

// Number of output rows path_gen allocates: sum over segments of ceil(duration * fs)
inline int64_t path_rows(const double* motion_def, int64_t segs, double fs) {
  int64_t total = 0;
  for (int64_t i = 0; i < segs; ++i) {
    if (motion_def[i * 9 + 7] < 0) return -1;
    total += static_cast<int64_t>(std::ceil(motion_def[i * 9 + 7] * fs));
  }
  return total;
}

// pathgen.path_gen.  motion_def [segs][9] (angles already in rad, NaN already 0, durations in
// seconds; NOT modified).  imu [cap][7], nav [cap][10], gps [cap][8] / odo [cap][5] (nullable).
// geomag_n [3]: geomagnetic field in the navigation frame [uT] (null: no magnetometer); mag [cap][4]
// gets (index, c_nb^T geomag_n) on every imu/nav row (pathgen.py:272-279).
// Returns the number of imu/nav rows (<= cap), or a negative error; *gps_rows gets the gps count.
inline int64_t path_gen(const double* ini, const double* motion_def, int64_t segs, double fs,
                        double osr, double fs_gps, double fs_odo, const double* mobility,
                        int ref_frame, int64_t cap, double* imu, double* nav, double* gps,
                        int64_t* gps_rows, double* odo, const double* geomag_n = nullptr,
                        double* mag = nullptr) {
  const double sim_freq = osr * fs;
  const double dt = 1.0 / sim_freq;
  const double alpha = 0.9, fa = alpha, fb = 1 - alpha;
  const double max_acc = mobility[0], max_dw = mobility[1], max_w = mobility[2];
  const double kp = 5.0, kd = 10.0;
  const double att_thr = 1e-4, vel_thr = 1e-4;
  const int64_t rows = path_rows(motion_def, segs, fs);
  if (rows < 0) return -2;
  if (rows == 0) return -3;
  if (rows > cap) return -4;
  const bool want_gps = gps != nullptr, want_odo = odo != nullptr;
  const bool want_mag = geomag_n != nullptr && mag != nullptr;
  const double gps_period = want_gps ? osr * std::nearbyint(fs / fs_gps) : 0.0;
  (void)fs_odo;  // the reference computes an odometer period but writes odo at the IMU rate

  double att_dot[3] = {0, 0, 0}, vel_dot_b[3] = {0, 0, 0};
  double acc_sum[3] = {0, 0, 0}, gyro_sum[3] = {0, 0, 0};
  double odo_dist = 0.0;
  double pos_n[3] = {ini[0], ini[1], ini[2]};
  double vel_b[3] = {ini[3], ini[4], ini[5]};
  double att[3] = {ini[6], ini[7], ini[8]};
  double c_nb[3][3];
  dcm_b2n(att, c_nb);
  double vel_n[3];
  mat_vec(c_nb, vel_b, vel_n);
  double pos_delta[3] = {0, 0, 0};
  const double g = geo_param(pos_n[0], pos_n[2]).g;
  if (ref_frame == 1) {
    double xyz[3];
    lla2ecef(pos_n, xyz);
    pos_n[0] = xyz[0];
    pos_n[1] = xyz[1];
    pos_n[2] = xyz[2];
  }
  double sim_count = 0.0;
  int64_t hi = 0, lo = 0;
  for (int64_t s = 0; s < segs; ++s) {
    const double* md = motion_def + s * 9;
    const long com_type = std::lround(md[0]);
    const double gps_vis = md[8];
    // parse_motion_def, pathgen.py:413-439
    double att_com[3], vel_com[3];
    const bool rel_att = (com_type == 3 || com_type == 5), rel_vel = (com_type == 3 || com_type == 4);
    for (int k = 0; k < 3; ++k) {
      att_com[k] = (rel_att ? att[k] : 0.0) + md[1 + k];
      vel_com[k] = (rel_vel ? vel_b[k] : 0.0) + md[4 + k];
    }
    if (com_type < 1 || com_type > 5) return -5;
    double att_filt[3] = {att[0], att[1], att[2]}, vel_filt[3] = {vel_b[0], vel_b[1], vel_b[2]};
    const double seg_end = sim_count + std::nearbyint(md[7] * fs * osr);   // python round(): half-even
    bool complete = false;
    while (sim_count < seg_end && !complete) {
      if (com_type == 1) {
        for (int k = 0; k < 3; ++k) {
          att_dot[k] = fa * att_dot[k] + fb * att_com[k];      // the commands are rates here
          vel_dot_b[k] = fa * vel_dot_b[k] + fb * vel_com[k];
        }
      } else {
        double e_att = 0, e_vel = 0;
        for (int k = 0; k < 3; ++k) {
          att_filt[k] = fa * att_filt[k] + fb * att_com[k];
          vel_filt[k] = fa * vel_filt[k] + fb * vel_com[k];
          vel_dot_b[k] = clampd((vel_filt[k] - vel_b[k]) / dt, max_acc);
          const double dd = clampd(kp * (att_com[k] - att[k]) + kd * (0 - att_dot[k]), max_dw);
          att_dot[k] = clampd(att_dot[k] + dd * dt, max_w);
          e_att += (att[k] - att_com[k]) * (att[k] - att_com[k]);
          e_vel += (vel_b[k] - vel_com[k]) * (vel_b[k] - vel_com[k]);
        }
        if (std::sqrt(e_att) < att_thr && std::sqrt(e_vel) < vel_thr) complete = true;
      }
      double pos_now[3] = {pos_n[0] + pos_delta[0], pos_n[1] + pos_delta[1], pos_n[2] + pos_delta[2]};
      double acc[3], gyro[3], pos_dot[3];
      true_sensor_output(pos_now, vel_b, att, c_nb, vel_dot_b, att_dot, ref_frame, g, acc, gyro, pos_dot);
      for (int k = 0; k < 3; ++k) {
        acc_sum[k] += acc[k];
        gyro_sum[k] += gyro[k];
      }
      if (py_mod(sim_count, osr) == 0.0) {
        if (hi >= cap) return -4;
        double* r = imu + hi * 7;
        r[0] = sim_count;
        for (int k = 0; k < 3; ++k) {
          r[1 + k] = acc_sum[k] / osr;
          r[4 + k] = gyro_sum[k] / osr;
          acc_sum[k] = gyro_sum[k] = 0.0;
        }
        double* v = nav + hi * 10;
        v[0] = sim_count;
        for (int k = 0; k < 3; ++k) {
          v[1 + k] = pos_n[k] + pos_delta[k];
          v[4 + k] = vel_n[k];
        }
        euler_range(att, v + 7);
        if (want_mag) {
          // c_nb^T geomag_n with the c_nb of this row's attitude.  The reference's c_nb.T.dot(geo_mag_n)
          // is NumPy's BLAS dgemv on a C-contiguous 3x3 matrix; OpenBLAS's x86-64 kernel rounds each row
          // as fma(a2, x2, fma(a0, x0, a1 x1)), and the same rounding here gives the same bits.
          double* b = mag + hi * 4;
          b[0] = sim_count;
          for (int k = 0; k < 3; ++k)
            b[1 + k] = std::fma(c_nb[2][k], geomag_n[2],
                                std::fma(c_nb[0][k], geomag_n[0], c_nb[1][k] * geomag_n[1]));
        }
        if (want_odo) {
          double* o = odo + hi * 5;
          o[0] = sim_count;
          o[1] = odo_dist;
          o[2] = vel_b[0];
          o[3] = vel_b[1];
          o[4] = vel_b[2];
        }
        ++hi;
      }
      if (want_gps && py_mod(sim_count, gps_period) == 0.0) {
        double* q = gps + lo * 8;
        q[0] = sim_count;
        for (int k = 0; k < 3; ++k) {
          q[1 + k] = pos_n[k] + pos_delta[k];
          q[4 + k] = vel_n[k];
        }
        q[7] = gps_vis;
        ++lo;
      }
      double speed2 = 0;
      for (int k = 0; k < 3; ++k) {
        pos_delta[k] = pos_delta[k] + pos_dot[k] * dt;
        speed2 += vel_b[k] * vel_b[k];
      }
      odo_dist = odo_dist + std::sqrt(speed2) * dt;
      for (int k = 0; k < 3; ++k) {
        vel_b[k] = vel_b[k] + vel_dot_b[k] * dt;
        att[k] = att[k] + att_dot[k] * dt;
      }
      dcm_b2n(att, c_nb);
      mat_vec(c_nb, vel_b, vel_n);
      sim_count += 1.0;
    }
    if (complete) {
      for (int k = 0; k < 3; ++k) att_dot[k] = vel_dot_b[k] = 0.0;
    }
  }
  if (gps_rows) *gps_rows = lo;
  return hi;
}

}  // namespace b2ins_host
