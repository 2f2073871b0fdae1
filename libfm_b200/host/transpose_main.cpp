// transpose_main.cpp -- drop-in for the reference's `transpose` tool (reference src/libfm/tools/transpose.cpp):
// a binary sparse matrix <ifile> (util/fmatrix.h:44-50, per row {uint size; size x {uint id; float value}})
// -> its transpose <ofile>, the .xt that -method mcmc|als read under -cache_size:
//   file_header {id = 2, float_size = 4, num_values, num_rows = the input's num_cols, num_cols = its num_rows},
//   then per column j {uint size; the (row, value) pairs naming j, in row order, a row's repeated j in entry order}.
// Same flags (-ifile, -ofile, -cache_size default 200000000, -help), byte-identical output.  Host memory is
// bounded by -cache_size as in the reference: one count per column, then one range of columns at a time whose
// entries fit cache_size / 2 bytes, each filled by one more read of the input.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>
#include <memory>
#include <string>
#include <vector>

#include "cli_flags.h"
#include "sparse_data.h"

namespace {

// The rows of a binary matrix, read in order through a FILE buffer.
class RowStream {
 public:
  RowStream(const std::string& path, const host::SparseData::XHeader& fh) : path_(path), fh_(fh) {
    f_ = fopen(path.c_str(), "rb");
    if (!f_) throw "could not open " + path;
    setvbuf(f_, nullptr, _IOFBF, 1 << 22);
    if (fseeko(f_, (off_t)sizeof(fh), SEEK_SET) != 0) throw "could not read " + path;
  }
  ~RowStream() { fclose(f_); }
  // fn(row, ids_and_values, size) for every row; every id must be below num_cols
  template <class F>
  void each(F fn) {
    uint64_t nnz = 0;
    for (uint32_t r = 0; r < fh_.num_rows; r++) {
      uint32_t size = 0;
      if (fread(&size, 4, 1, f_) != 1 || nnz + size > fh_.num_values) throw "could not read " + path_;
      buf_.resize(2 * (size_t)size);
      if (size && fread(buf_.data(), 8, size, f_) != size) throw "could not read " + path_;
      for (uint32_t i = 0; i < size; i++)
        if (buf_[2 * i] >= fh_.num_cols) throw "could not read " + path_ + ": row " + std::to_string(r) + " names column " + std::to_string(buf_[2 * i]) + " of " + std::to_string(fh_.num_cols);
      fn(r, buf_.data(), size);
      nnz += size;
    }
    if (nnz != fh_.num_values) throw "could not read " + path_;
  }

 private:
  std::string path_;
  host::SparseData::XHeader fh_;
  FILE* f_ = nullptr;
  std::vector<uint32_t> buf_;
};

}  // namespace

int main(int argc, char** argv) {
  try {
    host::CmdLine cmd(argc, argv);
    std::cout << "----------------------------------------------------------------------------" << std::endl;
    std::cout << "Transpose (libfm_b200)" << std::endl;
    std::cout << "----------------------------------------------------------------------------" << std::endl;
    const std::string p_ifile = cmd.add("ifile", "input file name, file has to be in binary sparse format [MANDATORY]");
    const std::string p_ofile = cmd.add("ofile", "output file name [MANDATORY]");
    const std::string p_cache = cmd.add("cache_size", "cache size for data storage, default=200000000");
    const std::string p_help = cmd.add("help", "this screen");
    if (cmd.has(p_help) || argc == 1) {
      cmd.print_help();
      return 0;
    }
    cmd.check();
    const std::string in_path = cmd.str(p_ifile), out_path = cmd.str(p_ofile);
    const uint64_t budget = (uint64_t)cmd.integer64(p_cache, 200000000) / 2;

    host::SparseData::XHeader fh;
    {
      std::ifstream in(in_path.c_str(), std::ios::binary);
      if (!in.is_open()) throw "could not open " + in_path;
      in.read(reinterpret_cast<char*>(&fh), sizeof(fh));
      if (!in || fh.id != 2 || fh.float_size != sizeof(float)) throw "could not read " + in_path;
      in.seekg(0, std::ios::end);
      const uint64_t fsize = (uint64_t)in.tellg();
      if (fsize != sizeof(fh) + 4ull * fh.num_rows + 8ull * fh.num_values) throw "could not read " + in_path;
    }
    std::cout << "num_rows=" << fh.num_rows << "\tnum_values=" << fh.num_values << "\tnum_features=" << fh.num_cols
              << std::endl;

    // (1) entries per column
    std::vector<uint64_t> per_col(fh.num_cols, 0);
    RowStream(in_path, fh).each([&](uint32_t, const uint32_t* e, uint32_t size) {
      for (uint32_t i = 0; i < size; i++) per_col[e[2 * i]]++;
    });

    // (2) ranges of columns whose .xt bytes fit the budget, each filled by one read of the input
    std::cout << "output to " << out_path << std::endl;
    std::ofstream out(out_path.c_str(), std::ios::out | std::ios::binary);
    if (!out.is_open()) throw "could not open " + out_path;
    const host::SparseData::XHeader oh = {2u, (uint32_t)sizeof(float), fh.num_values, fh.num_cols, fh.num_rows};
    out.write(reinterpret_cast<const char*>(&oh), sizeof(oh));
    std::vector<uint32_t> cache;  // per column of the range: {size; size x {row, value}}, as written
    std::vector<uint64_t> cursor;
    for (uint32_t lo = 0; lo < fh.num_cols;) {
      uint32_t hi = lo;
      uint64_t bytes = 0;
      while (hi < fh.num_cols && bytes + 4 + 8 * per_col[hi] <= budget) bytes += 4 + 8 * per_col[hi++];
      if (hi == lo)
        throw "column " + std::to_string(lo) + " of the transpose takes " + std::to_string(4 + 8 * per_col[lo]) +
            " bytes: -cache_size must be at least " + std::to_string(2 * (4 + 8 * per_col[lo]));
      cache.assign(bytes / 4, 0u);
      cursor.resize(hi - lo);
      uint64_t w = 0;
      for (uint32_t j = lo; j < hi; j++) {
        cache[w] = (uint32_t)per_col[j];
        cursor[j - lo] = w + 1;
        w += 1 + 2 * per_col[j];
      }
      RowStream(in_path, fh).each([&](uint32_t r, const uint32_t* e, uint32_t size) {
        for (uint32_t i = 0; i < size; i++) {
          const uint32_t j = e[2 * i];
          if (j < lo || j >= hi) continue;
          uint64_t& c = cursor[j - lo];
          cache[c] = r;
          cache[c + 1] = e[2 * i + 1];
          c += 2;
        }
      });
      out.write(reinterpret_cast<const char*>(cache.data()), (std::streamsize)bytes);
      lo = hi;
    }
    out.close();
    if (!out) throw "could not write " + out_path;
    return 0;
  } catch (std::string& e) {
    std::cerr << e << std::endl;
  } catch (char const*& e) {
    std::cerr << e << std::endl;
  } catch (const std::exception& e) {
    std::cerr << std::endl << "ERROR: " << e.what() << std::endl;
  }
  return 1;
}
