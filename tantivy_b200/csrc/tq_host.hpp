// What the library's host-only translation units (tq_plan.cpp, tq_multi.cpp, tq_writer.cpp) reach in the engine besides the C
// ABI: the thread-local last error that tq_last_error returns, and whether a prepared batch names a filter.  tq_engine.cu
// defines them.
#pragma once
#include <stdint.h>

#include <string>

#include "../../include/tantivy_b200.h"

namespace tq::host {

void set_last_error(const std::string& msg);
const std::string& last_error();
inline int fail(int code, const std::string& msg) {
  set_last_error(msg);
  return code;
}

// A batch prepared on c and not destroyed yet names filter_id (tq_filter_register / _unregister refuse it meanwhile).
bool filter_in_use(tq_ctx* c, uint32_t filter_id);

}  // namespace tq::host
