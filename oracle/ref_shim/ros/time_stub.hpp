// oracle/ref_shim/ros/time_stub.hpp — the ROS names the reference's A* search (front_end_Astar.hpp) touches for timing and
// logging only: ros::Time (now, difference, toSec), ROS_WARN / ROS_ERROR (no output).  Time is constant: no branch of the
// search depends on it.  Default constructions are counted: AstarGetSucc declares exactly three (`ros::Time t1,t2,t3;`,
// front_end_Astar.hpp:206) and nothing else default-constructs one, so count / 3 is the number of expanded nodes.
#pragma once
#include <cstdint>

namespace ros {
inline thread_local int64_t time_default_constructions = 0;
struct Duration {
    double sec{0.0};
    double toSec() const { return sec; }
};
struct Time {
    double sec{0.0};
    Time() { ++time_default_constructions; }
    static Time now() { return Time(0.0); }
    Duration operator-(const Time &o) const { return Duration{sec - o.sec}; }

  private:
    explicit Time(double s) : sec(s) {}
};
struct NodeHandle;
}  // namespace ros

#define ROS_WARN(...) ((void)0)
#define ROS_ERROR(...) ((void)0)
