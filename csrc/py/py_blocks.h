// SourceBlocks for Python (common/store_window.h): the description owns its slice addresses (a rebased one shares them);
// the ids and the selection are device pointers, or host pointers for the host loopback transport and resolve().
#pragma once
#include <memory>
#include <vector>

#include "common/store_window.h"

namespace bb {

struct PyBlocks {
  std::shared_ptr<const std::vector<uint64_t>> outer;
  SourceBlocks b;
};

}  // namespace bb
