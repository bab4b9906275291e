// Drop-in replacement for FASTER's SolverGurobi (reference faster/include/solverGurobi.hpp:61-186,
// faster/src/solverGurobi.cpp) with the optimiser behind it replaced by the GPU batch solver of libfaster_b200.so.
//
// Same class name, same public methods and public data members that Faster::replan() touches
// (faster.cpp:52-71,306-307,406-408,418,427,430,438,468,475,521-524,527,536-537,582-588), same meaning:
//   genNewTraj()  ascending factor sweep, FIRST feasible dt wins (solverGurobi.cpp:445-472); sets dt_,
//                 factor_that_worked_, trials_, runtime_ms_, sizes X_temp_ (resetX, :382-388)
//   fillX()       samples the solution every DC seconds into X_temp_ (:122-168)
// What differs:  one GPU launch evaluates every (factor x assignment) candidate of the sweep at once instead of one
// Gurobi MIQP per factor; the binaries b[t][p] (:217-246) are enumerated as interval->polytope assignments
// (all P^N of them while that is small -- the exact MIQP --, the non-decreasing ones beyond; see setAssignmentMode).  Methods that returned GRBLinExpr return the value of
// that expression at the current solution.  Additive: getCoeffs(), getCost(), getAssignment().
// Header-only; link with -lfaster_b200.  No Gurobi, no CPU fallback: if no GPU/context can be created genNewTraj()
// returns false and prints the reason (the reference's behaviour for every non-OPTIMAL status, :580-648).
#ifndef SOLVER_GUROBI_HPP
#define SOLVER_GUROBI_HPP

#include "faster_b200.h"
#if __has_include(<Eigen/Dense>)
#include <Eigen/Dense>             // the reference's faster_types.hpp relies on its includer for Eigen (solverGurobi.hpp:11 there)
#endif
#if __has_include("faster_types.hpp")
#include "faster_types.hpp"        // the reference's own `state` when this header lives in the reference tree
#else
#include "fq_state_compat.hpp"
#endif

#if __has_include(<decomp_geometry/polyhedron.h>)
#include <decomp_geometry/polyhedron.h>          // the reference's LinearConstraint3D, vec_Vecf (DecompUtil)
#else
#include "fq_compat.hpp"                         // look-alikes (adapts to Eigen when only Eigen is present)
#endif

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <iostream>
#include <vector>

// stands in for `mycallback : GRBCallback` (solverGurobi.hpp:50-59): only the abort flag survives
class mycallback
{
public:
  std::atomic<bool> should_terminate_{ false };
  mycallback() {}
  mycallback(const mycallback& o) : should_terminate_(o.should_terminate_.load()) {}
  mycallback& operator=(const mycallback& o) { should_terminate_ = o.should_terminate_.load(); return *this; }
};

class SolverGurobi
{
public:
  enum AssignmentMode { MONOTONE = 0, ALL = 1, AUTO = 2, EXACT = 3 };

  SolverGurobi()
  {
    v_max_ = 5; a_max_ = 3; j_max_ = 5;                       // solverGurobi.cpp:45-47
    for (int i = 0; i < 9; i++) x0_[i] = xf_[i] = 0;
  }
  ~SolverGurobi() { if (ctx_) fq_destroy(ctx_); }
  SolverGurobi(const SolverGurobi&) = delete;
  SolverGurobi& operator=(const SolverGurobi&) = delete;

  void setN(int N) { N_ = N; }                                                   // :60-63
  void createVars() { coeffs_.assign((size_t)12 * N_, 0.0); }                    // :70-84
  void setDC(double dc) { DC = dc; }                                             // :293-296
  void setBounds(double max_values[3])                                           // :409-416
  {
    v_max_ = max_values[0]; a_max_ = max_values[1]; j_max_ = max_values[2];
  }
  void setMaxConstraints() {}                                                    // limits are inputs of every solve
  void setForceFinalConstraint(bool f) { forceFinalConstraint_ = f; }            // :170-173
  void setFactorInitialAndFinalAndIncrement(double fi, double ff, double inc)    // :418-424
  {
    factor_initial_ = fi; factor_final_ = ff; factor_increment_ = inc;
  }
  void setVerbose(int v) { verbose_ = v; }                                       // :484-487
  void setThreads(int) {}                                                        // :479-482 (Gurobi threads: n/a)
  void setWMax(double w) { w_max_ = w; }                                         // :489-492
  void setMode(int mode) { mode_ = mode; }                                       // :65-68
  // declared in the reference (solverGurobi.hpp:100) but never defined there; kept so that code naming it still compiles
  void setDistances(vec_Vecf<3>& samples, std::vector<double> dist_near_obs) { (void)samples; (void)dist_near_obs; }
  void setDevice(int device) { device_ = device; devices_.clear(); releaseContext(); }   // additive: CUDA device index
  // additive: several GPUs for the batch entry points (fq_create_multi: the corridors of a batch are spread over the
  // devices, NCCL all-gather of the winners inside the library); genNewTraj() itself is one corridor and uses devices[0]
  void setDevices(const std::vector<int>& devices) { devices_ = devices; if (!devices.empty()) device_ = devices[0]; releaseContext(); }
  fq_ctx* context() { return ensureContext() ? ctx_ : nullptr; }                 // for the batch entry points of faster_b200.h
  // Which interval->polytope assignments are evaluated for every time allocation:
  //   ALL       every one of the P^N (the exact MIQP optimum, like Gurobi's branch-and-bound);
  //   MONOTONE  the non-decreasing ones only, C(N+P-1, P-1) (identical genNewTraj results in 960/960 measured sweeps,
  //             see DESIGN.md section 2);
  //   EXACT     branch-and-bound over all P^N on the GPU (fq_gen_new_traj_exact), ~125 us per sweep instead of ~80: the
  //             exact MIQP optimum, reported with exact = 1.  It falls back to the best non-decreasing assignment, reported
  //             with exact = 0, when the corridor has more than 2047 faces, when the tree's shared-memory footprint
  //             exceeds the GPU's (N = 16 safe: ~750 faces in one polytope), when a level of the tree has more than 65536
  //             open nodes, or when a node's solve gives up.  It refuses (FQ_E_ARG) when its non-decreasing pre-sweep is too
  //             long: C(N+P-1, N) > 2^20 (e.g. N = 10 with P >= 16) or C(N+P-1, N) x (time allocations) > 2^24;
  //   AUTO      (default) ALL while P^N <= auto_all_limit (4096: covers the shipped yaml, N=6 and <=3 polytopes: 729),
  //             EXACT beyond -- i.e. the reference's MIQP optimum within EXACT's limits.
  void setAssignmentMode(AssignmentMode m, long max_assignments = 16384, long auto_all_limit = 4096)
  {
    amode_ = m; max_sigma_ = max_assignments < 1 ? 1 : max_assignments; auto_all_limit_ = auto_all_limit;
    sig_N_ = -1;                                   // the cached assignment list depends on all three
  }

  void setX0(state& d)                                                           // :298-313
  {
    x0_[0] = d.pos.x(); x0_[1] = d.pos.y(); x0_[2] = d.pos.z();
    x0_[3] = d.vel.x(); x0_[4] = d.vel.y(); x0_[5] = d.vel.z();
    x0_[6] = d.accel.x(); x0_[7] = d.accel.y(); x0_[8] = d.accel.z();
  }
  void setXf(state& d)                                                           // :315-330
  {
    xf_[0] = d.pos.x(); xf_[1] = d.pos.y(); xf_[2] = d.pos.z();
    xf_[3] = d.vel.x(); xf_[4] = d.vel.y(); xf_[5] = d.vel.z();
    xf_[6] = d.accel.x(); xf_[7] = d.accel.y(); xf_[8] = d.accel.z();
  }
  void setPolytopes(std::vector<LinearConstraint3D> polytopes)                   // :175-178 (copy)
  {
    face_ofs_.assign(1, 0);
    Ab_.clear();
    for (size_t p = 0; p < polytopes.size(); p++)
    {
      const auto A = polytopes[p].A();
      const auto b = polytopes[p].b();
      for (int f = 0; f < (int)b.rows(); f++)
      {
        Ab_.push_back(A(f, 0)); Ab_.push_back(A(f, 1)); Ab_.push_back(A(f, 2)); Ab_.push_back(b(f));
      }
      face_ofs_.push_back(face_ofs_.back() + (int)b.rows());
    }
    P_ = (int)polytopes.size();
  }

  void StopExecution()                                                           // :30-34
  {
    cb_.should_terminate_ = true;
    std::cout << "Activated flag to stop execution" << std::endl;
  }
  void ResetToNormalState() { cb_.should_terminate_ = false; }                   // :36-39

  double getDTInitial() { return fq_dt_initial(x0_, xf_, lims(), N_); }          // :659-759
  void findDT(double factor) { dt_ = factor * std::max(getDTInitial(), 2 * DC); }  // :494-497
  void resetX()                                                                  // :382-388
  {
    X_temp_ = std::vector<state>((size_t)fq_num_samples(N_, dt_, DC));
  }

  bool genNewTraj()                                                              // :426-477
  {
    bool solved = false;
    trials_ = 0;
    if (factor_initial_ < 1) std::cout << "factor_initial_ is less than one, it doesn't make sense" << std::endl;
    runtime_ms_ = 0;
    // the factors the reference's loop would visit (same floating-point accumulation)
    std::vector<double> factors, dts;
    const double base = std::max(getDTInitial(), 2 * DC);
    for (double i = factor_initial_; i <= factor_final_ && cb_.should_terminate_ == false; i = i + factor_increment_)
    {
      factors.push_back(i);
      dts.push_back(i * base);
      if (factors.size() >= 4096) break;
    }
    if (!factors.empty())
    {
      const auto t0 = std::chrono::steady_clock::now();
      int dt_idx = -1, sig_idx = -1;
      int rc = FQ_E_NOGPU;
      const bool small_enum = std::pow((double)P_, (double)N_) <= (double)auto_all_limit_;
      if ((amode_ == EXACT || (amode_ == AUTO && !small_enum)) && P_ > 0)
      {
        if (ensureContext())
        {
          exact_sigma_.assign(N_, 0);
          rc = fq_gen_new_traj_exact(ctx_, N_, forceFinalConstraint_ ? 1 : 0, x0_, xf_, lims(), P_, face_ofs_.data(), Ab_.data(),
                                     (int)dts.size(), dts.data(), &dt_idx, exact_sigma_.data(), &cost_, coeffs_buf(), &bnb_nodes_,
                                     &bnb_exact_);
          sig_idx = -2;   // assignment held in exact_sigma_
        }
      }
      else if (ensureContext() && ensureAssignments())
        rc = fq_gen_new_traj(ctx_, N_, forceFinalConstraint_ ? 1 : 0, x0_, xf_, lims(), P_, face_ofs_.data(),
                             Ab_.empty() ? nullptr : Ab_.data(), (int)dts.size(), dts.data(), (int)n_sigma_,
                             sigmas_.empty() ? nullptr : sigmas_.data(), &dt_idx, &sig_idx, &cost_, coeffs_buf());
      runtime_ms_ = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
      temporal_ = temporal_ + 1;
      if (rc < 0 && !assignments_failed_)
        std::fprintf(stderr, "SolverGurobi(faster_b200): %s\n", ctx_ ? fq_last_error(ctx_) : fq_last_error(nullptr));
      assignments_failed_ = false;
      if (rc == 1)
      {
        solved = true;
        trials_ = dt_idx + 1;
        dt_ = dts[dt_idx];
        factor_that_worked_ = factors[dt_idx];
        sigma_idx_ = sig_idx;
      }
      else
      { // every factor was tried; dt_ stays at the last one, as in the reference
        trials_ = (int)factors.size();
        dt_ = dts.back();
      }
      resetX();
    }
    cb_.should_terminate_ = false;                                               // :474
    return solved;
  }
  bool callOptimizer() { return genNewTraj(); }                                  // :549-657 (kept for link-compat)

  void fillX()                                                                   // :122-168
  {
    const int n = (int)X_temp_.size();
    if (n == 0) return;
    std::vector<double> out((size_t)12 * n);
    fq_fill_x(N_, coeffs_.data(), dt_, DC, n, out.data());
    for (int i = 0; i < n; i++)
    {
      const double* o = &out[(size_t)12 * i];
      state s;
      s.setPos(o[0], o[1], o[2]); s.setVel(o[3], o[4], o[5]); s.setAccel(o[6], o[7], o[8]); s.setJerk(o[9], o[10], o[11]);
      X_temp_[i] = s;
    }
  }

  // model-building entry points of the reference: the model is implicit here, nothing to rebuild
  void setPolytopesConstraints() {}                                              // :180-291
  void setObjective() {}                                                         // :86-120
  void setConstraintsXf() {}                                                     // :332-357
  void setConstraintsX0() {}                                                     // :359-380
  void setDynamicConstraints() {}                                                // :499-524
  void setDistanceConstraints() {}                                               // declared only in the reference
  bool isWmaxSatisfied()                                                         // :527-547 (call is commented out at :459-462)
  {
    for (int n = 0; n < N_; n++)
    {
      const double xd = getVel(n, 0, 0), yd = getVel(n, 0, 1), xd2 = getAccel(n, 0, 0), yd2 = getAccel(n, 0, 1);
      const double num = xd * yd2 - yd * xd2, den = xd * xd + yd * yd;
      const double w_desired = (den > 0.001) ? std::fabs(num / den) : 0.5 * w_max_;
      if (w_desired > w_max_) return false;
    }
    return true;
  }

  // values of the reference's expression getters at the current solution (:761-862)
  double getPos(int t, double tau, int ii) const { const double* x = seg(t); return x[ii] * tau * tau * tau + x[3 + ii] * tau * tau + x[6 + ii] * tau + x[9 + ii]; }
  double getVel(int t, double tau, int ii) const { const double* x = seg(t); return 3 * x[ii] * tau * tau + 2 * x[3 + ii] * tau + x[6 + ii]; }
  double getAccel(int t, double tau, int ii) const { const double* x = seg(t); return 6 * x[ii] * tau + 2 * x[3 + ii]; }
  double getJerk(int t, double, int ii) const { return 6 * seg(t)[ii]; }
  double getA(int t, int ii) const { return seg(t)[ii]; }
  double getB(int t, int ii) const { return seg(t)[3 + ii]; }
  double getC(int t, int ii) const { return seg(t)[6 + ii]; }
  double getD(int t, int ii) const { return seg(t)[9 + ii]; }
  double getAn(int t, int ii) const { return seg(t)[ii] * dt_ * dt_ * dt_; }
  double getBn(int t, int ii) const { return seg(t)[3 + ii] * dt_ * dt_; }
  double getCn(int t, int ii) const { return seg(t)[6 + ii] * dt_; }
  double getDn(int t, int ii) const { return seg(t)[9 + ii]; }
  std::vector<double> getCP0(int t) const { return { getPos(t, 0, 0), getPos(t, 0, 1), getPos(t, 0, 2) }; }
  std::vector<double> getCP1(int t) const { return cp(t, 1); }
  std::vector<double> getCP2(int t) const { return cp(t, 2); }
  std::vector<double> getCP3(int t) const { return { getPos(t, dt_, 0), getPos(t, dt_, 1), getPos(t, dt_, 2) }; }

  // additive (north_star: "the returned coefficient matrix"): N x 12 row-major, x[t][i] order of solverGurobi.cpp:72
  const std::vector<double>& getCoeffs() const { return coeffs_; }
  double getCost() const { return cost_; }
  std::vector<int> getAssignment() const
  {
    std::vector<int> s;
    if (sigma_idx_ == -2)
      for (int t = 0; t < N_ && t < (int)exact_sigma_.size(); t++) s.push_back(exact_sigma_[t]);
    else if (sigma_idx_ >= 0 && !sigmas_.empty())
      for (int t = 0; t < N_; t++) s.push_back(sigmas_[(size_t)sigma_idx_ * N_ + t]);
    return s;
  }
  long getBnbNodes() const { return bnb_nodes_; }       // EXACT mode: nodes evaluated by the last sweep
  bool lastSweepExact() const { return bnb_exact_ != 0; }

  std::vector<state> X_temp_;
  double dt_ = 0;  // time step found by the solver
  int trials_ = 0;
  int temporal_ = 0;
  double runtime_ms_ = 0;
  double factor_that_worked_ = 0;
  int N_ = 10;
  mycallback cb_;

protected:
  const double* lims() { lim_[0] = v_max_; lim_[1] = a_max_; lim_[2] = j_max_; return lim_; }
  const double* seg(int t) const { return &coeffs_[(size_t)12 * t]; }
  double* coeffs_buf()
  {
    if (coeffs_.size() != (size_t)12 * N_) coeffs_.assign((size_t)12 * N_, 0.0);
    return coeffs_.data();
  }
  std::vector<double> cp(int t, int k) const
  {
    std::vector<double> r(3);
    for (int i = 0; i < 3; i++)
      r[i] = k == 1 ? (getCn(t, i) + 3 * getDn(t, i)) / 3 : (getBn(t, i) + 2 * getCn(t, i) + 3 * getDn(t, i)) / 3;
    return r;
  }
  bool ensureContext()
  {
    if (ctx_) return true;
    const int rc = devices_.size() > 1 ? fq_create_multi(&ctx_, (int)devices_.size(), devices_.data()) : fq_create(&ctx_, device_);
    // genNewTraj keeps the first feasible factor (solverGurobi.cpp:445-446): larger factors need not be evaluated
    if (rc == 0) fq_set_option(ctx_, "sweep_early_exit", 1);
    return rc == 0;
  }
  void releaseContext() { if (ctx_) { fq_destroy(ctx_); ctx_ = nullptr; } }
  // assignments enumerated for the current (N_, P_): rebuilt only when they change
  bool ensureAssignments()
  {
    if (P_ == 0) { sigmas_.clear(); n_sigma_ = 1; return true; }
    if (sig_N_ == N_ && sig_P_ == P_ && sig_mode_ == amode_) return true;
    sigmas_.clear();
    AssignmentMode mode = amode_;
    if (mode == AUTO || mode == EXACT) mode = std::pow((double)P_, (double)N_) <= (double)auto_all_limit_ ? ALL : MONOTONE;
    if (mode == MONOTONE)
    {
      const long total = fq_monotone_sigmas(N_, P_, nullptr, 0);
      std::vector<uint8_t> all((size_t)total * N_);
      fq_monotone_sigmas(N_, P_, all.data(), total);
      const long keep = std::min(total, max_sigma_);
      if (keep < total)                            // said once per (N, P, mode): a subset is not the reference's search space
        std::fprintf(stderr, "SolverGurobi(faster_b200): %ld monotone assignments, evaluating an even subset of %ld "
                             "(raise max_assignments, or use AUTO / EXACT for the exact MIQP optimum)\n", total, keep);
      for (long k = 0; k < keep; k++)
      {
        const long src = (keep == total || keep <= 1) ? k : (long)((double)k * (total - 1) / (keep - 1) + 0.5);
        sigmas_.insert(sigmas_.end(), all.begin() + (size_t)src * N_, all.begin() + (size_t)(src + 1) * N_);
      }
      n_sigma_ = keep;
    }
    else
    { // every assignment in P^N (only sensible for small P^N)
      double total = std::pow((double)P_, (double)N_);
      if (total > (double)max_sigma_)
      {
        std::fprintf(stderr, "SolverGurobi(faster_b200): P^N = %.0f assignments exceed max_assignments = %ld in ALL mode (use AUTO or EXACT)\n",
                     total, max_sigma_);
        assignments_failed_ = true;
        return false;
      }
      std::vector<uint8_t> s(N_, 0);
      for (;;)
      {
        sigmas_.insert(sigmas_.end(), s.begin(), s.end());
        int i = N_ - 1;
        while (i >= 0 && s[i] == P_ - 1) s[i--] = 0;
        if (i < 0) break;
        s[i]++;
      }
      n_sigma_ = (long)total;
    }
    sig_N_ = N_; sig_P_ = P_; sig_mode_ = amode_;
    return true;
  }

  double cost_ = 0;
  double xf_[3 * 3];
  double x0_[3 * 3];
  double v_max_, a_max_, j_max_;
  double lim_[3];
  double DC = 0.01;
  int P_ = 0;
  std::vector<int> face_ofs_{ 0 };
  std::vector<double> Ab_;           // rows [Ax Ay Az b]
  std::vector<double> coeffs_;       // N x 12
  std::vector<uint8_t> sigmas_, exact_sigma_;
  long bnb_nodes_ = 0;
  int bnb_exact_ = 1;
  long n_sigma_ = 1, max_sigma_ = 16384, auto_all_limit_ = 4096;
  int sig_N_ = -1, sig_P_ = -1, sig_mode_ = -1, sigma_idx_ = -1;
  AssignmentMode amode_ = AUTO;
  fq_ctx* ctx_ = nullptr;
  int device_ = 0;
  std::vector<int> devices_;
  bool assignments_failed_ = false;
  int verbose_ = 0;
  int mode_ = 0;
  bool forceFinalConstraint_ = true;
  double factor_initial_ = 2;
  double factor_final_ = 2;
  double factor_increment_ = 2;
  double w_max_ = 1;
};
#endif
