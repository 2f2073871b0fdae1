// xtblock_dump -- the block plan of a transposed file (host/sparse_data.h, BinaryBlocks::open_xt) and its
// reading through BlockReader, without a GPU, for tests/test_stream_mcmc_cpu.py.
//   xtblock_dump <stem> <cache_size> <out>
// prints "resident" when no <stem>.xt is streamed, else the plan line the command line prints and one
// "col_lo col_hi nnz offset" line per block; then reads every block (twice, as every pass restarts the reader)
// and writes its .xt bytes and its columns' sizes to <out>.xt and <out>.sizes.  Errors go to stderr as
// "ERROR: <text>", exit status 1.
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>

#include "sparse_data.h"

int main(int argc, char** argv) {
  if (argc != 4) {
    std::cerr << "usage: xtblock_dump <stem> <cache_size> <out>" << std::endl;
    return 2;
  }
  try {
    auto d = host::BinaryBlocks::open_xt(argv[1], strtoull(argv[2], nullptr, 10));
    if (!d) {
      std::cout << "resident" << std::endl;
      return 0;
    }
    d->print();
    for (const auto& b : d->blocks)
      std::cout << b.row_lo << " " << b.row_hi << " " << b.nnz << " " << b.offset << std::endl;
    host::BlockReader rd(*d, [](uint64_t n) { return malloc(n); }, [](void* p) { free(p); });
    const std::string out = argv[3];
    std::ofstream fx(out + ".xt", std::ios::binary), fs(out + ".sizes", std::ios::binary);
    for (int pass = 0; pass < 2; pass++) {
      rd.start();
      for (size_t b = 0; b < d->blocks.size(); b++) {
        const host::BlockReader::Buffer buf = rd.wait(b);
        const auto& bl = d->blocks[b];
        if (pass == 1) {
          fx.write(buf.x, (std::streamsize)bl.bytes());
          fs.write(reinterpret_cast<const char*>(buf.row_size), (std::streamsize)(4 * bl.rows()));
        }
        rd.release(b);
      }
      rd.stop();
    }
  } catch (const std::string& e) {
    std::cerr << "ERROR: " << e << std::endl;
    return 1;
  }
  return 0;
}
