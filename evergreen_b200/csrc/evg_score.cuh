// evg_score.cuh -- scalar arithmetic of the scheduler hot path, shared by every
// kernel.  Go semantics are reproduced exactly: int64 arithmetic wraps,
// time.Since saturates, Duration.Minutes()/Hours() are the stdlib two-term
// FP64 formulas, float->int conversions truncate (or floor where the reference
// calls math.Floor).  All FP64 operations use explicit round-to-nearest
// intrinsics on the device so nvcc cannot contract them into FMAs.
//
// Reference: scheduler/planner.go:209-337 (Unit.info, unitInfo.value,
// computeRankValue, computePriority), model/distro/distro.go:353-408 (factor
// getters), scheduler/utilization_based_host_allocator.go:268-296,324-409.
#pragma once
#include <stdint.h>

#include "../../include/evg_sched.h"

#if defined(__CUDACC__)
#define EVG_HD __host__ __device__ __forceinline__
#else
#define EVG_HD inline
#include <cmath>
#endif

namespace evg {

constexpr int64_t kSecond = 1000000000LL;
constexpr int64_t kMinute = 60 * kSecond;
constexpr int64_t kHour = 60 * kMinute;
constexpr int64_t kWeek = 7 * 24 * kHour;
constexpr int64_t kMaxDurationPerDistroHost = 30 * kMinute;  // globals.go:267
constexpr int64_t kI64Max = 0x7fffffffffffffffLL;
constexpr int64_t kI64Min = -kI64Max - 1;

// ---- FP64 with fixed rounding, never contracted ----
EVG_HD double fadd64(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  volatile double r = a + b;
  return r;
#endif
}
EVG_HD double fmul64(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  volatile double r = a * b;
  return r;
#endif
}
EVG_HD double fdiv64(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __ddiv_rn(a, b);
#else
  volatile double r = a / b;
  return r;
#endif
}
EVG_HD double i2d(int64_t x) {
#if defined(__CUDA_ARCH__)
  return __ll2double_rn(x);
#else
  return double(x);
#endif
}
EVG_HD int64_t d2i_trunc(double x) {  // Go int64(x)
#if defined(__CUDA_ARCH__)
  return __double2ll_rz(x);
#else
  return int64_t(x);
#endif
}
// Go leaves int64(x) of a NaN or of a value outside the int64 range implementation-defined; d2i_floor and d2i_ceil
// follow DESIGN.md §3: NaN gives 0 and a value beyond the range saturates at its end.  cvt.rmi / cvt.rpi saturate on
// their own; the NaN case is spelled out.
EVG_HD int64_t d2i_sat(double x) {  // x already integral
  if (x != x) return 0;
  if (x >= 9223372036854775808.0) return kI64Max;
  if (x < -9223372036854775808.0) return kI64Min;
  return int64_t(x);
}
EVG_HD int64_t d2i_floor(double x) {  // Go int64(math.Floor(x))
#if defined(__CUDA_ARCH__)
  return x != x ? 0 : __double2ll_rd(x);
#else
  return d2i_sat(std::floor(x));
#endif
}
EVG_HD int64_t d2i_ceil(double x) {  // Go int(math.Ceil(x))
#if defined(__CUDA_ARCH__)
  return x != x ? 0 : __double2ll_ru(x);
#else
  return d2i_sat(std::ceil(x));
#endif
}

// ---- Go integer / time semantics ----
EVG_HD int64_t wadd(int64_t a, int64_t b) { return int64_t(uint64_t(a) + uint64_t(b)); }
EVG_HD int64_t wsub(int64_t a, int64_t b) { return int64_t(uint64_t(a) - uint64_t(b)); }
EVG_HD int64_t wmul(int64_t a, int64_t b) { return int64_t(uint64_t(a) * uint64_t(b)); }

// time.Since(t) with a frozen clock; saturates like time.Time.Sub.
EVG_HD int64_t since(int64_t now, int64_t t) {
  if ((now | t) >= 0) return now - t;  // both non-negative: cannot overflow (EVG_TIME_ZERO is negative)
  if (t == EVG_TIME_ZERO) return kI64Max;
  const int64_t d = wsub(now, t);
  // signed overflow of now - t: operands differ in sign and the result's sign differs from now's
  if (((now ^ t) & (now ^ d)) < 0) return now < 0 ? kI64Min : kI64Max;
  return d;
}
// time.Duration.Minutes() / Hours()
EVG_HD double dur_minutes(int64_t d) { return fadd64(i2d(d / kMinute), fdiv64(i2d(d % kMinute), 60.0 * 1e9)); }
EVG_HD double dur_hours(int64_t d) { return fadd64(i2d(d / kHour), fdiv64(i2d(d % kHour), 60.0 * 60.0 * 1e9)); }

EVG_HD int64_t factor(int64_t x) { return x <= 0 ? 1 : x; }       // distro.go:353-408
EVG_HD double factor_d(double x) { return x <= 0.0 ? 1.0 : x; }  // distro.go:381-386

// unitInfo flags (planner.go:174-201)
enum : uint32_t {
  UF_MERGE_QUEUE = 1u,  // ContainsInCommitQueue
  UF_PATCH = 2u,        // ContainsInPatch
  UF_NON_GROUP = 4u,    // ContainsNonGroupTasks
  UF_GENERATE = 8u,     // ContainsGenerateTask
  UF_STEPBACK = 16u     // ContainsStepbackTask
};

// The reduction Unit.info performs over a unit's member tasks (planner.go:302-337).
struct UnitAcc {
  int64_t tiq;     // TimeInQueue
  int64_t rt;      // ExpectedRuntime
  int64_t max_p;   // MaxPriority (starts at 0)
  int64_t max_d;   // MaxNumDependents (starts at 0)
  int64_t n;       // len(TaskIDs)
  uint32_t flags;  // UF_*
};

EVG_HD void acc_init(UnitAcc& a) {
  a.tiq = 0; a.rt = 0; a.max_p = 0; a.max_d = 0; a.n = 0; a.flags = 0;
}

// One member task's contribution (planner.go:307-334).
EVG_HD void acc_add(UnitAcc& a, int64_t now, int32_t priority, int64_t expected_ns, int64_t queue_basis_ns,
                    int32_t num_dependents, int32_t group_id, uint32_t tflags) {
  uint32_t req = tflags & EVG_TF_REQ_MASK;
  if (req == EVG_TF_REQ_MERGE_QUEUE) a.flags |= UF_MERGE_QUEUE;
  else if (req == EVG_TF_REQ_PATCH) a.flags |= UF_PATCH;
  if (group_id < 0) a.flags |= UF_NON_GROUP;
  if (tflags & EVG_TF_GENERATE) a.flags |= UF_GENERATE;
  if (tflags & EVG_TF_STEPBACK) a.flags |= UF_STEPBACK;
  if (queue_basis_ns != EVG_TIME_ZERO) a.tiq = wadd(a.tiq, since(now, queue_basis_ns));
  if (int64_t(priority) > a.max_p) a.max_p = priority;
  a.rt = wadd(a.rt, expected_ns);
  if (int64_t(num_dependents) > a.max_d) a.max_d = num_dependents;
  a.n += 1;
}

// int64(math.Floor(d.Minutes() / float64(n))) and int64(d.Hours()) as the reference
// computes them (planner.go:230,239,256).  For small non-negative d the FP64 expression
// provably equals the integer quotient q: the fraction r/unit is at most 1 - 1/unit
// (1 - 1.7e-11 for minutes, 1 - 2.8e-13 for hours); below 2^15 minutes doubles are spaced
// 2^-38 = 3.6e-12 and below 2^10 hours 2^-43 = 1.1e-13, both finer than the gap to q + 1,
// so fl(q + frac) < q + 1 and floor/trunc give q; x / 1.0 == x exactly.  Everything else
// takes the literal FP64 path (tests/native/score_fastpath_check.cpp brute-forces this).
EVG_HD int64_t floor_minutes_over(int64_t d, int64_t n) {
  if (n == 1 && d >= 0 && d < (int64_t(1) << 15) * kMinute) return int64_t(uint64_t(d) / uint64_t(kMinute));
  return d2i_floor(fdiv64(dur_minutes(d), i2d(n)));
}
EVG_HD int64_t trunc_hours(int64_t d) {
  if (d >= 0 && d < (int64_t(1) << 10) * kHour) return int64_t(uint64_t(d) / uint64_t(kHour));
  return d2i_trunc(dur_hours(d));
}

// unitInfo.value (planner.go:209-300).  Returns TotalValue; when bd != nullptr
// also writes the 13-field breakdown (EVG_BD_*), bookkeeping quirks included.
EVG_HD int64_t unit_value(const UnitAcc& a, const evg_distro_cfg& c, int64_t* bd) {
  const int64_t len = a.n;
  const bool nongroup = (a.flags & UF_NON_GROUP) != 0;
  const bool gen = (a.flags & UF_GENERATE) != 0;
  const bool mq = (a.flags & UF_MERGE_QUEUE) != 0;
  const bool pat = (a.flags & UF_PATCH) != 0;
  // computePriority planner.go:271-300
  int64_t p_initial = wadd(1, a.max_p), p_tg = 0, p_gen = 0, p_cq = 0;
  int64_t prio = p_initial;
  if (!nongroup) { p_tg = len; prio = wadd(prio, len); }
  if (gen) {
    const int64_t gf = factor(c.generate_task_factor);
    const int64_t prev = prio;
    prio = wmul(prio, gf);
    p_gen = wsub(prio, prev);
    if (!nongroup) { p_tg = wmul(p_tg, gf); p_gen = wsub(p_gen, wmul(len, gf)); }
  }
  if (mq) { p_cq = 200; prio = wadd(prio, 200); }
  // computeRankValue planner.go:223-265
  int64_t r_patch = 0, r_patch_wait = 0, r_cq = 0, r_main = 0, r_step = 0;
  if (pat) {
    r_patch = factor(c.patch_factor);
    r_patch_wait = wmul(factor(c.patch_time_in_queue_factor), floor_minutes_over(a.tiq, len));
  } else if (mq) {
    r_cq = factor(c.commit_queue_factor);
  } else {
    const int64_t avg = len == 1 ? a.tiq : a.tiq / len;
    if (avg < kWeek) r_main = wmul(factor(c.mainline_time_in_queue_factor), trunc_hours(kWeek - avg));
    if (a.flags & UF_STEPBACK) r_step = factor(c.stepback_task_factor);
  }
  const int64_t r_deps = d2i_trunc(fmul64(factor_d(c.num_dependents_factor), i2d(a.max_d)));
  const int64_t r_rt = wmul(factor(c.expected_runtime_factor), floor_minutes_over(a.rt, len));
  int64_t rank = 1;
  rank = wadd(rank, r_patch); rank = wadd(rank, r_patch_wait); rank = wadd(rank, r_main);
  rank = wadd(rank, r_cq); rank = wadd(rank, r_step); rank = wadd(rank, r_deps); rank = wadd(rank, r_rt);
  const int64_t total = wadd(wmul(prio, rank), len);
  if (bd) {
    bd[EVG_BD_TASK_GROUP_LENGTH] = len; bd[EVG_BD_TOTAL_VALUE] = total;
    bd[EVG_BD_P_INITIAL] = p_initial; bd[EVG_BD_P_TASK_GROUP] = p_tg;
    bd[EVG_BD_P_GENERATOR] = p_gen; bd[EVG_BD_P_COMMIT_QUEUE] = p_cq;
    bd[EVG_BD_R_COMMIT_QUEUE] = r_cq; bd[EVG_BD_R_NUM_DEPENDENTS] = r_deps;
    bd[EVG_BD_R_ESTIMATED_RUNTIME] = r_rt; bd[EVG_BD_R_MAINLINE_WAIT] = r_main;
    bd[EVG_BD_R_STEPBACK] = r_step; bd[EVG_BD_R_PATCH] = r_patch; bd[EVG_BD_R_PATCH_WAIT] = r_patch_wait;
  }
  return total;
}

// Planner factors after the getters' "<= 0 -> 1" clamp (model/distro/distro.go:353-408),
// hoisted out of the per-task path.
struct PlannerFactors {
  int64_t patch, patch_tiq, commit_queue, mainline_tiq, runtime, generate, stepback;
  double num_dependents;
  int64_t nd_int;  // num_dependents as an integer when it is one (see single_task_value_fast), else 0
};
EVG_HD PlannerFactors clamp_factors(const evg_distro_cfg& c) {
  PlannerFactors f;
  f.patch = factor(c.patch_factor);
  f.patch_tiq = factor(c.patch_time_in_queue_factor);
  f.commit_queue = factor(c.commit_queue_factor);
  f.mainline_tiq = factor(c.mainline_time_in_queue_factor);
  f.runtime = factor(c.expected_runtime_factor);
  f.generate = factor(c.generate_task_factor);
  f.stepback = factor(c.stepback_task_factor);
  f.num_dependents = factor_d(c.num_dependents_factor);
  // an integral factor below 2^20 times a count below 2^31 is exact in FP64, so int64(f * float64(n)) == f * n
  f.nd_int = (f.num_dependents < 1048576.0 && f.num_dependents == i2d(d2i_trunc(f.num_dependents))) ? d2i_trunc(f.num_dependents) : 0;
  return f;
}

// unitInfo.value (planner.go:209-300) for the unit {one task that is not in a task group}:
// the common case, with len == 1 and ContainsNonGroupTasks folded in.  Same arithmetic as
// acc_add + unit_value; the parity tests compare both against the oracle.
EVG_HD int64_t single_task_value(const PlannerFactors& f, int64_t now, int32_t priority, int64_t expected_ns,
                                 int64_t queue_basis_ns, int32_t num_dependents, uint32_t tflags) {
  const uint32_t req = tflags & EVG_TF_REQ_MASK;
  const bool mq = req == EVG_TF_REQ_MERGE_QUEUE;
  const int64_t tiq = queue_basis_ns == EVG_TIME_ZERO ? 0 : since(now, queue_basis_ns);
  int64_t prio = wadd(1, priority > 0 ? int64_t(priority) : 0);
  if (tflags & EVG_TF_GENERATE) prio = wmul(prio, f.generate);
  if (mq) prio = wadd(prio, 200);
  int64_t term;
  if (req == EVG_TF_REQ_PATCH) {
    term = wadd(f.patch, wmul(f.patch_tiq, floor_minutes_over(tiq, 1)));
  } else if (mq) {
    term = f.commit_queue;
  } else {
    term = tiq < kWeek ? wmul(f.mainline_tiq, trunc_hours(wsub(kWeek, tiq))) : 0;
    if (tflags & EVG_TF_STEPBACK) term = wadd(term, f.stepback);
  }
  const int64_t r_deps = d2i_trunc(fmul64(f.num_dependents, i2d(num_dependents > 0 ? int64_t(num_dependents) : 0)));
  const int64_t r_rt = wmul(f.runtime, floor_minutes_over(expected_ns, 1));
  const int64_t rank = wadd(wadd(wadd(1, term), r_deps), r_rt);
  return wadd(wmul(prio, rank), 1);
}

// Straight-line form of single_task_value for the domain every production queue lives in:
//   clock and queue basis non-negative, 0 <= time in queue < 2^15 minutes (22.7 days) or no basis at all,
//   0 <= expected runtime < 2^15 minutes, integral NumDependentsFactor (f.nd_int != 0).
// There Minutes()/Hours() are exact integer quotients (see floor_minutes_over / trunc_hours; whole hours of
// d are whole minutes of d over 60), time.Since cannot saturate and the FP64 dependents term is an exact
// product, so the value is the same integer -- without a data-dependent branch.  Callers test the domain for
// a whole warp at once (score_fast_domain) and fall back to single_task_value otherwise;
// tests/native/score_fastpath_check.cpp compares the two on random in-domain inputs.
constexpr uint64_t kFastLimit = uint64_t(int64_t(1) << 15) * uint64_t(kMinute);
EVG_HD bool score_fast_domain(int64_t now, int64_t expected_ns, int64_t queue_basis_ns) {  // requires now >= 0
  const bool q_ok = queue_basis_ns == EVG_TIME_ZERO || (queue_basis_ns >= 0 && uint64_t(now - queue_basis_ns) < kFastLimit);
  return q_ok && uint64_t(expected_ns) < kFastLimit;
}
EVG_HD int64_t single_task_value_fast(const PlannerFactors& f, int64_t now, int32_t priority, int64_t expected_ns,
                                      int64_t queue_basis_ns, int32_t num_dependents, uint32_t tflags) {
  const uint32_t req = tflags & EVG_TF_REQ_MASK;
  const bool mq = req == EVG_TF_REQ_MERGE_QUEUE, pat = req == EVG_TF_REQ_PATCH;
  const uint64_t tiq = queue_basis_ns == EVG_TIME_ZERO ? 0ull : uint64_t(now - queue_basis_ns);
  int64_t prio = int64_t(1u + uint32_t(priority > 0 ? priority : 0));
  prio = wmul(prio, (tflags & EVG_TF_GENERATE) ? f.generate : 1);
  prio = wadd(prio, mq ? 200 : 0);
  const uint64_t left = tiq < uint64_t(kWeek) ? uint64_t(kWeek) - tiq : 0ull;  // mainline: what is left of the first week
  const uint32_t mins = uint32_t((pat ? tiq : left) / uint64_t(kMinute));
  const uint32_t qty = pat ? mins : mins / 60u;  // patch: whole minutes waited; mainline: whole hours left
  int64_t term = wmul(pat ? f.patch_tiq : f.mainline_tiq, int64_t(qty));
  term = wadd(term, pat ? f.patch : ((tflags & EVG_TF_STEPBACK) ? f.stepback : 0));
  if (mq) term = f.commit_queue;
  const int64_t r_deps = wmul(f.nd_int, int64_t(uint32_t(num_dependents > 0 ? num_dependents : 0)));
  const int64_t r_rt = wmul(f.runtime, int64_t(uint32_t(uint64_t(expected_ns) / uint64_t(kMinute))));
  const int64_t rank = wadd(wadd(wadd(1, term), r_deps), r_rt);
  return wadd(wmul(prio, rank), 1);
}

// 32-bit form of single_task_value_fast: when, in addition to the straight-line domain, every planner factor is
// below 2^14 (config_scheduler.go:132-159 validates them to 0..100) and the task's priority and NumDependents are
// below 2^15, every intermediate fits 32 bits:
//   prio = (1 + p) * gen + 200            < 2^15 * 2^14 + 200     < 2^30
//   rank = 1 + f*qty + f + nd*d + rt*min  < 1 + 2^29 + 2^14 + 2^29 + 2^29 < 2^31
// so TotalValue = prio * rank + 1 is ONE 32x32->64 multiply-add and cannot wrap.  Same integer as unit_value
// (tests/native/score_fastpath_check.cpp compares them); everything else takes the 64-bit forms above.
constexpr int64_t kFactor32Limit = int64_t(1) << 14;
constexpr uint32_t kTask32Limit = 1u << 15;
struct Factors32 {
  uint32_t patch, patch_tiq, commit_queue, mainline_tiq, runtime, generate, stepback, nd;
  uint32_t ok;       // distro-wide preconditions hold (clock non-negative, all factors small, integral NumDependentsFactor)
  uint32_t ok_base;  // the same without the NumDependentsFactor condition: callers that tabulate int64(factor * n) for small n
};
EVG_HD Factors32 factors32(const PlannerFactors& f, int64_t now) {
  Factors32 g;
  g.patch = uint32_t(f.patch); g.patch_tiq = uint32_t(f.patch_tiq); g.commit_queue = uint32_t(f.commit_queue);
  g.mainline_tiq = uint32_t(f.mainline_tiq); g.runtime = uint32_t(f.runtime); g.generate = uint32_t(f.generate);
  g.stepback = uint32_t(f.stepback); g.nd = uint32_t(f.nd_int);
  g.ok_base = now >= 0 && f.patch < kFactor32Limit && f.patch_tiq < kFactor32Limit &&
              f.commit_queue < kFactor32Limit && f.mainline_tiq < kFactor32Limit && f.runtime < kFactor32Limit &&
              f.generate < kFactor32Limit && f.stepback < kFactor32Limit;
  g.ok = g.ok_base && f.nd_int != 0 && f.nd_int < kFactor32Limit;
  return g;
}
// per-task part of the domain (requires Factors32::ok): score_fast_domain plus small priority / dependents
EVG_HD bool score32_domain(int64_t now, int32_t priority, int32_t num_dependents, int64_t expected_ns, int64_t queue_basis_ns) {
  return score_fast_domain(now, expected_ns, queue_basis_ns) && priority < int32_t(kTask32Limit) &&
         num_dependents < int32_t(kTask32Limit);
}
// NumDependentsFactor need not be integral for the 32-bit form: int64(factor * float64(n)) (planner.go:247) is tabulated
// per distro for n < kNdTable (nearly every task) by nd_table_entry; entries must stay below 2^29 like the products above.
constexpr int kNdTable = 64;
constexpr uint32_t kNdTermLimit = 1u << 29;
EVG_HD int64_t nd_table_entry(const PlannerFactors& f, int n) { return d2i_trunc(fmul64(f.num_dependents, i2d(n))); }
// domain of single_task_value32_nd: everything score32_domain checks except NumDependents (the caller resolved its term)
EVG_HD bool score32_domain_nd(int64_t now, int32_t priority, int64_t expected_ns, int64_t queue_basis_ns) {
  return score_fast_domain(now, expected_ns, queue_basis_ns) && priority < int32_t(kTask32Limit);
}
// The kernels' form of that test, one OR of everything that must be small (nonzero = outside): time in queue and expected
// duration below 2^50 ns (13 days, inside kFastLimit; with now >= 0 -- Factors32::ok_base -- a wrapped now - t below 2^50
// is the exact difference, so a basis before 1970 needs no test of its own), priority below 2^15, the resolved
// NumDependents term below 2^29 (kNdTermLimit; "not representable" is 0xFFFFFFFF).
EVG_HD uint32_t score32_bad(int64_t now, int32_t priority, int64_t expected_ns, int64_t queue_basis_ns, uint32_t nd_term) {
  const uint64_t tiq = queue_basis_ns == EVG_TIME_ZERO ? 0ull : uint64_t(now - queue_basis_ns);
  return uint32_t((tiq | uint64_t(expected_ns)) >> 50) | (uint32_t(priority > 0 ? priority : 0) >> 15) | (nd_term >> 29);
}
EVG_HD uint64_t single_task_value32_nd(const Factors32& f, int64_t now, int32_t priority, int64_t expected_ns,
                                       int64_t queue_basis_ns, uint32_t nd_term, uint32_t tflags) {
  const uint32_t req = tflags & EVG_TF_REQ_MASK;
  const bool mq = req == EVG_TF_REQ_MERGE_QUEUE, pat = req == EVG_TF_REQ_PATCH;
  const uint64_t tiq = queue_basis_ns == EVG_TIME_ZERO ? 0ull : uint64_t(now - queue_basis_ns);
  const uint32_t p = 1u + uint32_t(priority > 0 ? priority : 0);
  const uint32_t prio = p * ((tflags & EVG_TF_GENERATE) ? f.generate : 1u) + (mq ? 200u : 0u);
  const uint64_t left = tiq < uint64_t(kWeek) ? uint64_t(kWeek) - tiq : 0ull;
  const uint32_t mins = uint32_t((pat ? tiq : left) / uint64_t(kMinute));
  const uint32_t qty = pat ? mins : mins / 60u;
  uint32_t term = (pat ? f.patch_tiq : f.mainline_tiq) * qty + (pat ? f.patch : ((tflags & EVG_TF_STEPBACK) ? f.stepback : 0u));
  if (mq) term = f.commit_queue;
  const uint32_t rank = 1u + term + nd_term + f.runtime * uint32_t(uint64_t(expected_ns) / uint64_t(kMinute));
  return uint64_t(prio) * uint64_t(rank) + 1ull;
}
EVG_HD uint64_t single_task_value32(const Factors32& f, int64_t now, int32_t priority, int64_t expected_ns,
                                    int64_t queue_basis_ns, int32_t num_dependents, uint32_t tflags) {
  const uint32_t req = tflags & EVG_TF_REQ_MASK;
  const bool mq = req == EVG_TF_REQ_MERGE_QUEUE, pat = req == EVG_TF_REQ_PATCH;
  const uint64_t tiq = queue_basis_ns == EVG_TIME_ZERO ? 0ull : uint64_t(now - queue_basis_ns);
  const uint32_t p = 1u + uint32_t(priority > 0 ? priority : 0);
  const uint32_t prio = p * ((tflags & EVG_TF_GENERATE) ? f.generate : 1u) + (mq ? 200u : 0u);
  const uint64_t left = tiq < uint64_t(kWeek) ? uint64_t(kWeek) - tiq : 0ull;  // mainline: what is left of the first week
  const uint32_t mins = uint32_t((pat ? tiq : left) / uint64_t(kMinute));
  const uint32_t qty = pat ? mins : mins / 60u;  // patch: whole minutes waited; mainline: whole hours left
  uint32_t term = (pat ? f.patch_tiq : f.mainline_tiq) * qty + (pat ? f.patch : ((tflags & EVG_TF_STEPBACK) ? f.stepback : 0u));
  if (mq) term = f.commit_queue;
  const uint32_t rank = 1u + term + f.nd * uint32_t(num_dependents > 0 ? num_dependents : 0) +
                        f.runtime * uint32_t(uint64_t(expected_ns) / uint64_t(kMinute));
  return uint64_t(prio) * uint64_t(rank) + 1ull;
}

// Sort-key encoding: ascending unsigned order of enc_value(v) == descending v.
EVG_HD uint64_t enc_value(int64_t v) { return ~(uint64_t(v) ^ 0x8000000000000000ULL); }
EVG_HD int64_t dec_value(uint64_t k) { return int64_t((~k) ^ 0x8000000000000000ULL); }

// Canonical tie word: anchor of the unit the task is emitted from (smallest
// input index among the unit's primary members -- unique per unit), then the
// task's rank inside that unit; 21 bits each (distros hold < 2^21 tasks).
constexpr int kIdxBits = 21;
constexpr int64_t kMaxTasksPerDistro = (int64_t(1) << kIdxBits) - 1;
EVG_HD uint64_t enc_tie(uint32_t anchor, uint32_t rank_in_unit) {
  return (uint64_t(anchor) << kIdxBits) | uint64_t(rank_in_unit);
}

// TaskList.Less (planner.go:387-405) extended by input index: true when task x
// sorts strictly before task y inside a unit.
EVG_HD bool in_unit_less(int32_t tgo_x, int32_t nd_x, int32_t pr_x, int64_t ex_x, uint32_t ix,
                         int32_t tgo_y, int32_t nd_y, int32_t pr_y, int64_t ex_y, uint32_t iy) {
  if (tgo_x != tgo_y) return tgo_x < tgo_y;
  if (nd_x != nd_y) return nd_x > nd_y;
  if (pr_x != pr_y) return pr_x > pr_y;
  if (ex_x != ex_y) return ex_x > ex_y;
  return ix < iy;
}

// calcNewHostsNeeded (utilization_based_host_allocator.go:268-296)
EVG_HD int64_t calc_new_hosts_needed(int64_t short_ns, int64_t threshold, int64_t exp_free, int64_t n_long,
                                     int64_t n_overdue, int64_t n_mq, bool round_down) {
  double x = fdiv64(i2d(short_ns), i2d(threshold));
  x = fadd64(x, -i2d(exp_free));
  x = fadd64(x, i2d(n_long));
  x = fadd64(x, i2d(n_overdue));
  x = fadd64(x, i2d(n_mq));
  if (exp_free < 1 && x > 0.0 && x < 1.0) return 1;
  int64_t n = round_down ? d2i_floor(x) : d2i_ceil(x);
  return n < 0 ? 0 : n;
}

// One running host's contribution to getSoonToBeFreeHosts (allocator.go:357-378),
// already scaled by futureHostFraction.
EVG_HD double soon_free_term(int64_t now, int64_t expected, int64_t stddev, int64_t start, int64_t threshold,
                             double future_host_fraction) {
  const int64_t elapsed = since(now, start);
  const int64_t left = wsub(expected, elapsed);
  double f;
  if (elapsed > kMaxDurationPerDistroHost && stddev > 0 && elapsed > wadd(expected, wmul(3, stddev))) f = 0.0;
  else f = fdiv64(i2d(wsub(threshold, left)), i2d(threshold));
  if (f < 0.0) f = 0.0;
  if (f > 1.0) f = 1.0;
  return fmul64(future_host_fraction, f);
}

// isMaxHostsCapacity (allocator.go:397-409)
EVG_HD bool is_max_hosts_capacity(int64_t max_hosts, bool pool, int64_t pool_max, int64_t n_new, int64_t n_existing) {
  if (pool && n_new > wsub(wmul(max_hosts, pool_max), n_existing)) return true;  // Go int: wraps
  return n_new + n_existing > max_hosts;
}

}  // namespace evg
