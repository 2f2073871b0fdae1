// The launch plan of one SGDA epoch (libfm_b200/csrc/fm_sgda_plan.h) for tests/test_sgda_plan_cpu.py.
// stdin: "N V lambda_steps", then the training blocks' first rows and row count on one line (empty: resident),
// then the validation blocks' likewise.  stdout: one launch per line, "h_begin h_end vc0 train_block val_block
// moments".
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "fm_sgda_plan.h"

static std::vector<uint32_t> read_lo(std::istream& in) {
  std::string line;
  std::getline(in, line);
  std::istringstream s(line);
  std::vector<uint32_t> lo;
  for (uint32_t x; s >> x;) lo.push_back(x);
  return lo;
}

int main() {
  uint64_t n = 0, v = 0;
  int lam = 0;
  std::string line;
  std::getline(std::cin, line);
  std::istringstream(line) >> n >> v >> lam;
  const std::vector<uint32_t> tl = read_lo(std::cin), vl = read_lo(std::cin);
  const uint64_t nbt = tl.empty() ? 0 : tl.size() - 1, nbv = vl.empty() ? 0 : vl.size() - 1;
  for (const fmb::SgdaLaunch& l : fmb::sgda_plan(n, v, lam != 0, tl.data(), nbt, vl.data(), nbv))
    std::printf("%llu %llu %llu %lld %lld %d\n", (unsigned long long)l.h_begin, (unsigned long long)l.h_end,
                (unsigned long long)l.vc0, (long long)l.train_block, (long long)l.val_block, (int)l.moments);
  return 0;
}
