// dep_shim.h — what the reference's DependenciesInJob (CtldPublicDefs.h:413-428) and
// DependenciesInJob::update (CtldPublicDefs.cpp:144-159) need around them.
// TEST INFRASTRUCTURE ONLY (oracle/ rules).
//
//  * absl::Time / absl::Duration as int64 seconds with Abseil's infinities at both ends:
//    InfinitePast() / InfiniteFuture() are INT64_MIN / INT64_MAX, and Time + Duration
//    keeps an infinite time infinite and saturates on overflow, as Abseil does.
//  * crane::grpc::DependencyType (PublicDefs.proto:136-141).
//  * CRANE_ERROR counts the calls instead of logging.
#pragma once
#include <algorithm>
#include <cstdint>
#include <limits>
#include <unordered_map>
#include <utility>

namespace absl {

class Duration {
 public:
  constexpr Duration() = default;
  static constexpr Duration FromSeconds(int64_t s) { Duration d; d.s_ = s; return d; }
  constexpr int64_t seconds() const { return s_; }
 private:
  int64_t s_{0};
};
template <class T>
constexpr Duration Seconds(T n) { return Duration::FromSeconds(static_cast<int64_t>(n)); }

class Time {
 public:
  constexpr Time() = default;
  static constexpr Time FromUnix(int64_t s) { Time t; t.s_ = s; return t; }
  constexpr int64_t unix_seconds() const { return s_; }
  friend constexpr bool operator<(Time a, Time b) { return a.s_ < b.s_; }
  friend constexpr bool operator<=(Time a, Time b) { return a.s_ <= b.s_; }
  friend constexpr bool operator>=(Time a, Time b) { return a.s_ >= b.s_; }
  friend constexpr bool operator==(Time a, Time b) { return a.s_ == b.s_; }
 private:
  int64_t s_{0};
};
constexpr Time InfinitePast() { return Time::FromUnix(std::numeric_limits<int64_t>::min()); }
constexpr Time InfiniteFuture() { return Time::FromUnix(std::numeric_limits<int64_t>::max()); }
inline Time operator+(Time t, Duration d) {
  if (t == InfinitePast() || t == InfiniteFuture()) return t;
  int64_t r;
  if (__builtin_add_overflow(t.unix_seconds(), d.seconds(), &r)) return d.seconds() > 0 ? InfiniteFuture() : InfinitePast();
  return Time::FromUnix(r);
}

}  // namespace absl

namespace crane::grpc {
enum DependencyType { AFTER = 0, AFTER_ANY = 1, AFTER_OK = 2, AFTER_NOT_OK = 3 };
}  // namespace crane::grpc

using job_id_t = uint32_t;

inline thread_local uint32_t g_crane_error_calls = 0;
#define CRANE_ERROR(...) (++g_crane_error_calls)
