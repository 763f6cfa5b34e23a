// Host-side controller of the probability-flow ODE sampler (SURVEY.md §8f-4).
//
// The reference integrates the reverse ODE with scipy.integrate.solve_ivp(method='RK45') and moves the whole state
// through host numpy for every right-hand-side evaluation (/root/reference/sgmse/sampling/__init__.py:117-141).  The
// integrator is third-party (scipy, pinned 1.10.1 in requirements_version.txt:14; 1.18.1 in this image): its published
// algorithm -- Dormand & Prince 5(4) with the step-size control of Hairer, Norsett & Wanner, "Solving Ordinary
// Differential Equations I", Sec. II.4, in the form of scipy/integrate/_ivp/rk.py (RungeKutta._step_impl, rk_step),
// common.py (select_initial_step, norm) and base.py (OdeSolver.step) -- is restated here as a scalar state machine.
// All vector work goes through `Ops`, so the same controller drives the CUDA kernels of the sampler (engine.cu:
// OdeDeviceOps -- only ONE double per norm crosses the PCIe bus) and a plain host callback
// (sgmse_b200_rk45_host, CPU-tested against scipy itself in tests/test_cabi_host.py).
//
// Ops contract (y: current state, K[0..6]: stage derivatives, "stage": the argument of the next evaluation):
//   size_t size()                                            number of (complex) unknowns
//   void   combine(int s, const double* a, double h, bool to_new)
//                                                            stage = y + (sum_{j<s} a[j] K[j]) * h ; to_new: y_new = stage
//   void   eval(double t, int slot)                          K[slot] = f(t, stage)
//   double norm_init(int which, double rtol, double atol)    rms(v / (atol + |y| rtol)), v = y | K[0] | K[1] - K[0]
//   double norm_err(const double* E, double h, double rtol, double atol)
//                                                            rms((sum_{j<7} E[j] K[j]) * h / (atol + max(|y|, |y_new|) rtol))
//   void   accept()                                          y = y_new, K[0] = K[6]   (first-same-as-last)
#pragma once
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstddef>
#include <vector>

namespace sgmse {
namespace rk45 {

constexpr int kStages = 6;
constexpr double C[6] = {0.0, 1.0 / 5, 3.0 / 10, 4.0 / 5, 8.0 / 9, 1.0};
constexpr double A[6][5] = {
    {0, 0, 0, 0, 0},
    {1.0 / 5, 0, 0, 0, 0},
    {3.0 / 40, 9.0 / 40, 0, 0, 0},
    {44.0 / 45, -56.0 / 15, 32.0 / 9, 0, 0},
    {19372.0 / 6561, -25360.0 / 2187, 64448.0 / 6561, -212.0 / 729, 0},
    {9017.0 / 3168, -355.0 / 33, 46732.0 / 5247, 49.0 / 176, -5103.0 / 18656}};
constexpr double B[6] = {35.0 / 384, 0, 500.0 / 1113, 125.0 / 192, -2187.0 / 6784, 11.0 / 84};
constexpr double E[7] = {-71.0 / 57600, 0, 71.0 / 16695, -71.0 / 1920, 17253.0 / 339200, -22.0 / 525, 1.0 / 40};
constexpr double kSafety = 0.9, kMinFactor = 0.2, kMaxFactor = 10.0;
constexpr double kErrorExponent = -1.0 / 5.0;   // -1 / (error_estimator_order + 1), error_estimator_order = 4

struct Result {
  double t = 0;       // time reached
  int nfev = 0;       // right-hand-side evaluations (what the reference returns as `nfe`)
  int steps = 0;      // accepted steps
  int rejected = 0;   // rejected step attempts
  int status = 0;     // 0: reached t_bound; -1: required step size below the spacing of doubles (scipy's "failed");
                      // -2: max_attempts exhausted; -3: non-finite error norm or step size.  -2 / -3 are not scipy states:
                      // with a NaN right-hand side scipy's loop never terminates (h_abs becomes NaN and every comparison
                      // is false); here the solve stops and reports it
};

// The controller as a resumable per-system state machine.  next(v) returns the next request of the solve; v is the
// value of the previous request when that was a norm (ignored otherwise).  A request's `accept` flag asks for
// accept() (y = y_new, K[0] = K[6]) before the request itself, also before kDone.  solve() below is one stepper on
// one Ops; solve_groups() advances many in lockstep.  The arithmetic is that of scipy's RK45 in the order it runs.
struct Request {
  enum Kind { kEval, kNorm, kDone } kind = kDone;
  int s = 0;                 // kEval: combine(s, a, h, to_new), then eval(t, slot s);  kNorm: which (0..2 norm_init, 3 norm_err)
  const double* a = nullptr; // kEval: combination coefficients;  kNorm 3: E
  double h = 0, t = 0;
  bool to_new = false;
  bool accept = false;
};

class Stepper {
 public:
  Stepper(size_t size, double t0, double t_bound, double rtol, double atol, int max_attempts)
      : size_(size), t0_(t0), t_bound_(t_bound), rtol_(rtol < 100 * DBL_EPSILON ? 100 * DBL_EPSILON : rtol),   // validate_tol
        atol_(atol), max_attempts_(max_attempts), direction_(t_bound != t0 ? (t_bound > t0 ? 1.0 : -1.0) : 1.0), t_(t0) {}

  double rtol() const { return rtol_; }
  double atol() const { return atol_; }
  const Result& result() const { return r_; }

  Request next(double v) {
    Request q;
    switch (pc_) {
      case kStart:
        pc_ = kAfterF0;
        return eval(0, nullptr, 0.0, false, t_);                             // self.f = fun(t0, y0)
      case kAfterF0: {                                                       // ---- select_initial_step ----
        const double interval = std::fabs(t_bound_ - t0_);
        if (size_ == 0) h_abs_ = INFINITY;
        else if (interval == 0.0) h_abs_ = 0.0;
        else { pc_ = kD0; return norm(0, nullptr, 0.0); }
        return step_top(false);
      }
      case kD0: d0_ = v; pc_ = kD1; return norm(1, nullptr, 0.0);
      case kD1: {
        d1_ = v;
        h0_ = (d0_ < 1e-5 || d1_ < 1e-5) ? 1e-6 : 0.01 * d0_ / d1_;
        h0_ = std::min(h0_, std::fabs(t_bound_ - t0_));
        pc_ = kY1;
        return eval(1, &kOne, h0_ * direction_, false, t0_ + h0_ * direction_);   // y1 = y0 + h0 * direction * f0
      }
      case kY1: pc_ = kD2; return norm(2, nullptr, 0.0);
      case kD2: {
        const double d2 = v / h0_;
        const double h1 = (d1_ <= 1e-15 && d2 <= 1e-15) ? std::max(1e-6, h0_ * 1e-3) : std::pow(0.01 / std::max(d1_, d2), 1.0 / 5.0);
        h_abs_ = std::min(std::min(100 * h0_, h1), std::fabs(t_bound_ - t0_));
        return step_top(false);
      }
      case kStage:                                                           // rk_step
        if (++s_ < kStages) return eval(s_, A[s_], h_, false, t_ + C[s_] * h_);
        if (s_ == kStages) return eval(kStages, B, h_, true, t_ + h_);
        pc_ = kErr;
        return norm(3, E, h_);
      case kErr: {
        const double err = v;
        if (!std::isfinite(err) && !(err > 0)) { nonfinite_ = true; return step_end(); }   // NaN (inf just rejects the step)
        if (err < 1) {
          double factor = err == 0 ? kMaxFactor : std::min(kMaxFactor, kSafety * std::pow(err, kErrorExponent));
          if (rejected_) factor = std::min(1.0, factor);
          h_abs_ *= factor;
          accepted_ = true;
        } else {
          // err = +inf: pow() gives 0 and the step shrinks by MIN_FACTOR, like Python's max(0.2, 0.0)
          const double f = kSafety * std::pow(err, kErrorExponent);
          h_abs_ *= (kMinFactor < f) ? f : kMinFactor;
          rejected_ = true;
          ++r_.rejected;
        }
        return attempt();
      }
      case kFinished: break;
    }
    return q;
  }

 private:
  enum Pc { kStart, kAfterF0, kD0, kD1, kY1, kD2, kStage, kErr, kFinished };
  static constexpr double kOne = 1.0;

  Request eval(int s, const double* a, double h, bool to_new, double t) {
    Request q;
    q.kind = Request::kEval; q.s = s; q.a = a; q.h = h; q.to_new = to_new; q.t = t;
    ++r_.nfev;
    return q;
  }
  Request norm(int which, const double* a, double h) {
    Request q;
    q.kind = Request::kNorm; q.s = which; q.a = a; q.h = h;
    return q;
  }
  Request done(int status, bool accept) {
    r_.status = status;
    r_.t = t_;
    pc_ = kFinished;
    Request q;
    q.accept = accept;
    return q;
  }
  // ---- OdeSolver.step until finished: one step, preceded by the accept() of the previous one ----
  Request step_top(bool accept) {
    if (size_ == 0 || t_ == t_bound_) { t_ = t_bound_; return done(0, accept); }
    min_step_ = 10 * std::fabs(std::nextafter(t_, direction_ * INFINITY) - t_);
    if (h_abs_ < min_step_) h_abs_ = min_step_;                              // (max_step = inf)
    accepted_ = rejected_ = failed_ = exhausted_ = false;
    nonfinite_ = !std::isfinite(h_abs_);
    t_new_ = t_;
    Request q = attempt();
    if (accept) q.accept = true;
    return q;
  }
  Request attempt() {                                                        // while (!accepted && !nonfinite)
    if (accepted_ || nonfinite_) return step_end();
    if (h_abs_ < min_step_) { failed_ = true; return step_end(); }
    if (attempts_ >= max_attempts_) { exhausted_ = true; return step_end(); }
    ++attempts_;
    double h = h_abs_ * direction_;
    t_new_ = t_ + h;
    if (direction_ * (t_new_ - t_bound_) > 0) t_new_ = t_bound_;
    h = t_new_ - t_;
    h_abs_ = std::fabs(h);
    h_ = h;
    s_ = 1;
    pc_ = kStage;
    return eval(1, A[1], h_, false, t_ + C[1] * h_);
  }
  Request step_end() {
    if (nonfinite_) return done(-3, false);
    if (failed_) return done(-1, false);
    if (exhausted_) return done(-2, false);
    ++r_.steps;
    t_ = t_new_;
    if (direction_ * (t_ - t_bound_) >= 0) return done(0, true);
    return step_top(true);
  }

  size_t size_;
  double t0_, t_bound_, rtol_, atol_;
  int max_attempts_;
  double direction_, t_;
  Pc pc_ = kStart;
  Result r_;
  double d0_ = 0, d1_ = 0, h0_ = 0, h_abs_ = 0, h_ = 0, t_new_ = 0, min_step_ = 0;
  int s_ = 0, attempts_ = 0;
  bool accepted_ = false, rejected_ = false, failed_ = false, exhausted_ = false, nonfinite_ = false;
};

template <class Ops>
Result solve(Ops& ops, double t0, double t_bound, double rtol, double atol, int max_attempts) {
  Stepper sp(ops.size(), t0, t_bound, rtol, atol, max_attempts);
  double v = 0.0;
  for (;;) {
    const Request q = sp.next(v);
    if (q.accept) ops.accept();
    if (q.kind == Request::kDone) return sp.result();
    if (q.kind == Request::kEval) {
      ops.combine(q.s, q.a, q.h, q.to_new);
      ops.eval(q.t, q.s);
    } else {
      v = q.s == 3 ? ops.norm_err(q.a, q.h, sp.rtol(), sp.atol()) : ops.norm_init(q.s, sp.rtol(), sp.atol());
    }
  }
}

// Lockstep driver: `systems` independent solves, at most `slots` of them in flight.  Each round serves the pending
// request of every system in flight -- all norms in one ops.norms() call, then all evaluations in one ops.evals()
// call -- and then advances each stepper.  A finished system frees its slot, and the next unstarted system takes it:
// its first evaluation is served in the following round.  Every system sees exactly the requests, in exactly the
// order, that solve() would issue for it alone, so its result does not depend on the others.
//
// GroupOps contract (slot: 0..slots-1, the buffers a system in flight owns):
//   size_t size(int sys)
//   void   start(int sys, int slot)                       y(slot) = the initial state of system `sys`
//   void   norms(int n, const int* slot, const Request* q, double rtol, double atol, double* out)
//                                                         out[i] = the norm q[i] asks of slot[i]
//   void   evals(int n, const int* sys, const int* slot, const Request* q)
//                                                         for each i: combine then eval q[i] on slot[i]
//   void   accept(int slot)
//   void   finish(int sys, int slot, const Result& r)     the system's final y leaves slot `slot`
// Returns the number of rounds.
template <class GroupOps>
long long solve_groups(GroupOps& ops, int systems, int slots, double t0, double t_bound, double rtol, double atol,
                       int max_attempts, Result* results) {
  struct Slot { int sys = -1; Stepper sp{0, 0, 0, 0, 0, 0}; Request q; double v = 0; };
  std::vector<Slot> sl((size_t)std::max(1, std::min(slots, systems)));
  int next_sys = 0;
  auto advance = [&](Slot& s, int k) {
    for (;;) {
      s.q = s.sp.next(s.v);
      if (s.q.accept) ops.accept(k);
      if (s.q.kind != Request::kDone) return;
      results[s.sys] = s.sp.result();
      ops.finish(s.sys, k, s.sp.result());
      s.sys = -1;
      if (next_sys >= systems) return;
      s.sys = next_sys++;                                                  // refill
      s.sp = Stepper(ops.size(s.sys), t0, t_bound, rtol, atol, max_attempts);
      s.v = 0;
      ops.start(s.sys, k);
    }
  };
  for (int k = 0; k < (int)sl.size(); ++k) {
    if (next_sys >= systems) break;
    sl[k].sys = next_sys++;
    sl[k].sp = Stepper(ops.size(sl[k].sys), t0, t_bound, rtol, atol, max_attempts);
    ops.start(sl[k].sys, k);
    advance(sl[k], k);
  }
  std::vector<int> sys_ids, slot_ids;
  std::vector<Request> reqs;
  const Stepper tol(0, t0, t_bound, rtol, atol, max_attempts);              // the validated tolerances every stepper uses
  std::vector<double> vals;
  long long rounds = 0;
  for (;;) {
    bool any = false;
    for (const Slot& s : sl) any = any || s.sys >= 0;
    if (!any) return rounds;
    ++rounds;
    slot_ids.clear(); reqs.clear();
    for (int k = 0; k < (int)sl.size(); ++k)
      if (sl[k].sys >= 0 && sl[k].q.kind == Request::kNorm) { slot_ids.push_back(k); reqs.push_back(sl[k].q); }
    if (!slot_ids.empty()) {
      vals.assign(slot_ids.size(), 0.0);
      ops.norms((int)slot_ids.size(), slot_ids.data(), reqs.data(), tol.rtol(), tol.atol(), vals.data());
      for (size_t i = 0; i < slot_ids.size(); ++i) sl[slot_ids[i]].v = vals[i];
    }
    sys_ids.clear(); slot_ids.clear(); reqs.clear();
    for (int k = 0; k < (int)sl.size(); ++k)
      if (sl[k].sys >= 0 && sl[k].q.kind == Request::kEval) { sys_ids.push_back(sl[k].sys); slot_ids.push_back(k); reqs.push_back(sl[k].q); }
    if (!slot_ids.empty()) ops.evals((int)slot_ids.size(), sys_ids.data(), slot_ids.data(), reqs.data());
    for (int k = 0; k < (int)sl.size(); ++k)
      if (sl[k].sys >= 0) advance(sl[k], k);
  }
}

}  // namespace rk45
}  // namespace sgmse
