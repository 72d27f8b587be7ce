// Minimal stand-in for <boost/bind.hpp> (not installed here) so FullSystem::linearizeAll compiles unmodified: its
// multi-thread branch binds linearizeAll_Reductor for IndexThreadReduce, which the harness never runs
// (multiThreading = false).  Test infrastructure only (oracle/ref_build_linearize.mk).
#pragma once
#include <functional>
namespace boost {
using std::bind;
}  // namespace boost
using std::placeholders::_1;
using std::placeholders::_2;
using std::placeholders::_3;
using std::placeholders::_4;
