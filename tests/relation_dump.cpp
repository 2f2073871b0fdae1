// Test helper: run the CLI's relation loaders (RelationData, RelationJoin in libfm_b200/host/sparse_data.h) on one
// block and dump what they read as raw little-endian arrays.  Built on the fly by tests/test_relation_cli_cpu.py.
//   relation_dump <stem> <train cases> <test cases> <out>
// out: u64 num_cases, num_feature, num_groups, nnz; u64 col_ptr[num_feature + 1]; u32 row[nnz]; f32 val[nnz];
//      u32 attr_group[num_feature]; u32 train join[train cases]; u32 test join[test cases]
#include <cstdio>
#include <iostream>
#include <sstream>
#include "sparse_data.h"

int main(int argc, char** argv) {
  if (argc != 5) return 2;
  host::RelationData d;
  host::RelationJoin join[2];
  std::ostringstream sink;
  std::streambuf* saved = std::cout.rdbuf(sink.rdbuf());
  try {
    d.load(argv[1]);
    join[0].load(std::string(argv[1]) + ".train", std::stoull(argv[2]));
    join[1].load(std::string(argv[1]) + ".test", std::stoull(argv[3]));
  } catch (std::string& e) {
    std::cout.rdbuf(saved);
    std::cerr << "ERROR: " << e << std::endl;
    return 1;
  }
  std::cout.rdbuf(saved);
  FILE* f = fopen(argv[4], "wb");
  const uint64_t head[4] = {d.num_cases, d.num_feature, d.num_groups, d.row.size()};
  fwrite(head, 8, 4, f);
  fwrite(d.col_ptr.data(), 8, d.col_ptr.size(), f);
  fwrite(d.row.data(), 4, d.row.size(), f);
  fwrite(d.val.data(), 4, d.val.size(), f);
  fwrite(d.attr_group.data(), 4, d.attr_group.size(), f);
  for (const host::RelationJoin& j : join) fwrite(j.rows.data(), 4, j.rows.size(), f);
  fclose(f);
  return 0;
}
