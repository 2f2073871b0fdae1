// xblock_dump -- the block plan and the block reader of host/sparse_data.h without a GPU (plain host
// memory stands in for the page-locked buffers), for tests/test_stream_cpu.py.
//   xblock_dump <stem> <cache_size> <out>
// prints "resident" when the data set is loaded whole, else one "row_lo row_hi nnz offset" line per block;
// then reads every block through BlockReader and writes, per block, its .x bytes, its rows' sizes and its
// targets to <out>.x, <out>.sizes and <out>.y.  Errors go to stderr as "ERROR: <text>", exit status 1.
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>

#include "sparse_data.h"

int main(int argc, char** argv) {
  if (argc != 4) {
    std::cerr << "usage: xblock_dump <stem> <cache_size> <out>" << std::endl;
    return 2;
  }
  try {
    auto d = host::BinaryBlocks::open(argv[1], strtoull(argv[2], nullptr, 10));
    if (!d) {
      std::cout << "resident" << std::endl;
      return 0;
    }
    for (const auto& b : d->blocks)
      std::cout << b.row_lo << " " << b.row_hi << " " << b.nnz << " " << b.offset << std::endl;
    host::BlockReader rd(*d, [](uint64_t n) { return malloc(n); }, [](void* p) { free(p); });
    const std::string out = argv[3];
    std::ofstream fx(out + ".x", std::ios::binary), fs(out + ".sizes", std::ios::binary), fy(out + ".y", std::ios::binary);
    for (int pass = 0; pass < 2; pass++) {  // a second pass restarts the reader, as every epoch does
      rd.start();
      for (size_t b = 0; b < d->blocks.size(); b++) {
        const host::BlockReader::Buffer buf = rd.wait(b);
        const auto& bl = d->blocks[b];
        if (pass == 1) {
          fx.write(buf.x, (std::streamsize)bl.bytes());
          fs.write(reinterpret_cast<const char*>(buf.row_size), (std::streamsize)(4 * bl.rows()));
          fy.write(reinterpret_cast<const char*>(buf.target), (std::streamsize)(4 * bl.rows()));
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
