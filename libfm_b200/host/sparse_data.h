// sparse_data.h -- the host-side sparse loader of the drop-in command line.
//
// Produces the SoA CSR that libfmb200 consumes (row offsets, column ids, values,
// targets) from the inputs the reference's Data::load accepts (reference
// src/libfm/src/Data.h:113-290):
//   * libfm text:  `target id:value id:value ...`  (# comments, blank lines)
//   * binary pair: <file>.x + <file>.y (or .data + .target), the format the
//     reference's `convert` tool writes (src/libfm/tools/convert.cpp:143-198,
//     util/fmatrix.h:44-50, util/matrix.h:364-380)
// Ordering (rows in file order, entries in line order) and the derived numbers
// (num_feature = max id + 1, min/max target) are bit-exact contracts.  Text files are
// parsed by all host cores (the reference: two sscanf passes on one core).  A binary pair
// larger than -cache_size is not loaded whole: BinaryBlocks plans its blocks and
// BlockReader reads them, one pass at a time.
#pragma once
#include <algorithm>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <limits>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

namespace host {

struct SparseData {
  std::vector<uint64_t> row_ptr{0};
  std::vector<uint32_t> col;
  std::vector<float> val;
  std::vector<float> target;
  int num_feature = 0;
  float min_target = +std::numeric_limits<float>::max();
  float max_target = -std::numeric_limits<float>::max();

  uint64_t num_cases() const { return row_ptr.size() - 1; }
  uint64_t num_values() const { return row_ptr.back(); }

  static bool file_exists(const std::string& f) {
    std::ifstream in(f.c_str());
    return in.is_open();
  }

  // Data::load (Data.h:113-290).  Prints the same progress lines.
  void load(const std::string& filename) {
    std::cout << "has x = " << 1 << std::endl;
    std::cout << "has xt = " << 0 << std::endl;
    std::string fx, fy;
    if (binary_pair(filename, &fx, &fy)) {
      load_binary(fx, fy);
    } else {
      load_text(filename);
    }
  }

  // text input only (the `convert` tool never looks for binary siblings of its input)
  void load_text_file(const std::string& filename) { load_text(filename); }

  // libfm.cpp:302-303
  void binarize_targets() {
    for (auto& t : target) t = (t <= 0.0f) ? -1.0f : 1.0f;
  }

 private:
  static std::string parse_error(const std::string& line, char at) {
    return "cannot parse line \"" + line + "\" at character " + at;
  }

  // One contiguous piece of the file, parsed by one thread.
  struct TextChunk {
    std::vector<uint64_t> row_end;  // entries so far after each row (chunk-local)
    std::vector<uint32_t> col;
    std::vector<float> val, target;
    int max_id = 0;
    bool has_feature = false;
    float min_target = +std::numeric_limits<float>::max();
    float max_target = -std::numeric_limits<float>::max();
    std::string error;  // first parse error of the chunk, in file order
  };

  // Parse the lines in [begin, end) (each made NUL-terminated in place).  Same grammar
  // as Data::load (Data.h:192-225): "%f" then repeated "%d:%f", '#' comments.
  static void parse_chunk(char* begin, char* end, TextChunk& out) {
    char* line = begin;
    while (line < end) {
      char* nl = static_cast<char*>(memchr(line, '\n', (size_t)(end - line)));
      char* line_end = nl ? nl : end;
      *line_end = 0;
      const char* p = line;
      while (*p == ' ' || *p == '\t') p++;
      if (*p != 0 && *p != '#') {  // Data.h:200-201: blank and comment lines are skipped
        char* e0 = nullptr;
        const float y = strtof(p, &e0);  // "%f"
        if (e0 == p) {
          out.error = parse_error(line, p[0]);
          return;
        }
        p = e0;
        out.target.push_back(y);
        if (y < out.min_target) out.min_target = y;
        if (y > out.max_target) out.max_target = y;
        for (;;) {
          // "%d:%f" -- %d skips white space, ':' must follow the digits directly,
          // %f skips white space again
          const char* q = p;
          while (*q == ' ' || *q == '\t') q++;
          char* e1 = nullptr;
          const long id = strtol(q, &e1, 10);
          if (e1 == q || *e1 != ':') break;
          char* e2 = nullptr;
          const float x = strtof(e1 + 1, &e2);
          if (e2 == e1 + 1) break;
          out.col.push_back((uint32_t)(int)id);
          out.val.push_back(x);
          if ((int)id > out.max_id) out.max_id = (int)id;
          out.has_feature = true;
          p = e2;
        }
        while (*p == ' ' || *p == '\t') p++;
        if (*p != 0 && *p != '#') {  // Data.h:218-220
          out.error = parse_error(line, p[0]);
          return;
        }
        out.row_end.push_back(out.col.size());
      }
      line = line_end + 1;
    }
  }

  // The reference parses the file twice with sscanf on one core (Data.h:180-290) and
  // that dominates its wall time on large inputs (SURVEY.md section 8 a9).  Here the
  // file is read once, cut at line boundaries and parsed by all host cores; the chunks
  // are concatenated in file order, so the CSR is identical to the sequential result.
  void load_text(const std::string& filename) {
    std::string buf;
    {
      std::ifstream in(filename.c_str(), std::ios::binary);
      if (!in.is_open()) throw "unable to open " + filename;
      in.seekg(0, std::ios::end);
      const std::streamoff len = in.tellg();
      in.seekg(0, std::ios::beg);
      buf.resize((size_t)(len > 0 ? len : 0) + 1);
      if (len > 0) in.read(&buf[0], len);
      buf[buf.size() - 1] = 0;
    }
    char* base = &buf[0];
    char* stop = base + buf.size() - 1;
    unsigned hw = std::thread::hardware_concurrency();
    size_t n_chunks = hw ? hw : 4;
    if (n_chunks > 32) n_chunks = 32;
    if ((size_t)(stop - base) < (1u << 20)) n_chunks = 1;  // small files: not worth a thread
    std::vector<char*> cut(n_chunks + 1);
    cut[0] = base;
    cut[n_chunks] = stop;
    for (size_t i = 1; i < n_chunks; i++) {
      char* guess = base + (size_t)(stop - base) * i / n_chunks;
      if (guess < cut[i - 1]) guess = cut[i - 1];
      char* nl = static_cast<char*>(memchr(guess, '\n', (size_t)(stop - guess)));
      cut[i] = nl ? nl + 1 : stop;
    }
    std::vector<TextChunk> chunks(n_chunks);
    std::vector<std::thread> workers;
    for (size_t i = 1; i < n_chunks; i++)
      workers.emplace_back(parse_chunk, cut[i], cut[i + 1], std::ref(chunks[i]));
    parse_chunk(cut[0], cut[1], chunks[0]);
    for (auto& w : workers) w.join();

    uint64_t rows = 0, entries = 0;
    for (const auto& c : chunks) {
      if (!c.error.empty()) throw c.error;  // the first error in file order
      rows += c.target.size();
      entries += c.col.size();
    }
    row_ptr.assign(1, 0);
    row_ptr.reserve(rows + 1);
    col.resize(entries);
    val.resize(entries);
    target.resize(rows);
    bool has_feature = false;
    int max_id = 0;
    uint64_t r0 = 0, e0 = 0;
    for (const auto& c : chunks) {
      for (uint64_t re : c.row_end) row_ptr.push_back(e0 + re);
      if (!c.col.empty()) {
        memcpy(&col[e0], c.col.data(), c.col.size() * sizeof(uint32_t));
        memcpy(&val[e0], c.val.data(), c.val.size() * sizeof(float));
      }
      if (!c.target.empty()) memcpy(&target[r0], c.target.data(), c.target.size() * sizeof(float));
      r0 += c.target.size();
      e0 += c.col.size();
      has_feature |= c.has_feature;
      if (c.max_id > max_id) max_id = c.max_id;
      if (c.min_target < min_target) min_target = c.min_target;
      if (c.max_target > max_target) max_target = c.max_target;
    }
    num_feature = has_feature ? max_id + 1 : 0;  // Data.h:227-229
    std::cout << "num_rows=" << num_cases() << "\tnum_values=" << num_values()
              << "\tnum_features=" << num_feature << "\tmin_target=" << min_target
              << "\tmax_target=" << max_target << std::endl;
  }

 public:
  // file_header of a binary matrix (util/fmatrix.h:44-50)
  struct XHeader {
    uint32_t id, float_size;
    uint64_t num_values;
    uint32_t num_rows, num_cols;
  };
  static_assert(sizeof(XHeader) == 24, "file_header layout (util/fmatrix.h:44-50)");

  // target vector: {uint version=1, uint type_size=4, uint n} + float[n]  (matrix.h:364-380)
  static std::vector<float> read_targets(const std::string& fy) {
    std::ifstream in(fy.c_str(), std::ios::binary);
    uint32_t hdr[3];
    in.read(reinterpret_cast<char*>(hdr), sizeof(hdr));
    if (!in || hdr[0] != 1 || hdr[1] != sizeof(float)) throw "could not read " + fy;
    std::vector<float> t(hdr[2]);
    in.read(reinterpret_cast<char*>(t.data()), sizeof(float) * (size_t)hdr[2]);
    if (!in) throw "could not read " + fy;
    return t;
  }

  // The header of fx, checked against the n_rows targets of fy (no check when fy is empty); leaves `in` at the
  // first row.  transposed: fx is a .xt, whose columns are the cases.
  static XHeader read_header(std::ifstream& in, const std::string& fx, const std::string& fy, uint64_t n_rows,
                             bool transposed = false) {
    if (!in.is_open()) throw "could not open " + fx;
    XHeader fh;
    in.read(reinterpret_cast<char*>(&fh), sizeof(fh));
    if (!in || fh.id != 2 || fh.float_size != sizeof(float)) throw "could not read " + fx;
    if (!fy.empty() && (transposed ? fh.num_cols : fh.num_rows) != n_rows)
      throw std::string(transposed ? "case count of " : "row count of ") + fx + " and " + fy + " differ";
    // a truncated / corrupt header must not size the arrays: bound num_values by the file
    in.seekg(0, std::ios::end);
    const uint64_t fsize = (uint64_t)in.tellg();
    in.seekg(sizeof(fh), std::ios::beg);
    const uint64_t fixed = sizeof(fh) + 4ull * fh.num_rows;
    if (!in || fsize < fixed || fh.num_values > (fsize - fixed) / 8) throw "could not read " + fx;
    return fh;
  }

  // The binary pair Data::load reads for `filename` (.data + .target, else .x + .y); false for text input.
  static bool binary_pair(const std::string& filename, std::string* fx, std::string* fy) {
    for (const char* const* e : {data_target_, x_y_}) {
      if (file_exists(filename + e[0]) && file_exists(filename + e[1])) {
        *fx = filename + e[0];
        *fy = filename + e[1];
        return true;
      }
    }
    return false;
  }

 private:
  static constexpr const char* data_target_[2] = {".data", ".target"};
  static constexpr const char* x_y_[2] = {".x", ".y"};

 public:
  // The binary matrix fx -- file_header (24 B), then per row {uint size; size x {uint id; float value}} -- into
  // row_ptr, col and val (a .x, or a .xt whose rows are the features); fy and n_rows as in read_header
  static XHeader read_matrix(const std::string& fx, const std::string& fy, uint64_t n_rows, bool transposed,
                             std::vector<uint64_t>& row_ptr, std::vector<uint32_t>& col, std::vector<float>& val) {
    std::ifstream in(fx.c_str(), std::ios::binary);
    const XHeader fh = read_header(in, fx, fy, n_rows, transposed);
    col.resize(fh.num_values);
    val.resize(fh.num_values);
    row_ptr.assign(1, 0);
    row_ptr.reserve((size_t)fh.num_rows + 1);
    std::vector<char> buf;
    uint64_t pos = 0;
    for (uint32_t r = 0; r < fh.num_rows; r++) {
      uint32_t size = 0;
      in.read(reinterpret_cast<char*>(&size), sizeof(size));
      if (!in || pos + size > fh.num_values) throw "could not read " + fx;
      buf.resize((size_t)size * 8);
      in.read(buf.data(), buf.size());
      if (!in) throw "could not read " + fx;
      for (uint32_t j = 0; j < size; j++) {
        memcpy(&col[pos + j], buf.data() + 8 * (size_t)j, 4);
        memcpy(&val[pos + j], buf.data() + 8 * (size_t)j + 4, 4);
      }
      pos += size;
      row_ptr.push_back(pos);
    }
    if (pos != fh.num_values) throw "could not read " + fx;
    return fh;
  }

 private:
  void load_binary(const std::string& fx, const std::string& fy) {
    target = read_targets(fy);
    std::cout << "data... ";
    num_feature = (int)read_matrix(fx, fy, target.size(), false, row_ptr, col, val).num_cols;
    for (float y : target) {  // Data.h:166-171
      if (y < min_target) min_target = y;
      if (y > max_target) max_target = y;
    }
    std::cout << "num_cases=" << num_cases() << "\tnum_values=" << num_values()
              << "\tnum_features=" << num_feature << "\tmin_target=" << min_target
              << "\tmax_target=" << max_target << std::endl;
  }
};

// DataMetaInfo::loadGroupsFromFile (Data.h:84-96), the rules of -meta and of a relation block's .groups: one group
// id per attribute, read with >>, where a value the file lacks reads as 0.  group holds the n attributes' groups on
// return; the result is the group count, 1 + the largest id.
inline uint32_t read_groups(const std::string& file, uint32_t n, std::vector<uint32_t>& group) {
  std::ifstream in(file.c_str());
  if (!in.is_open()) throw "Unable to open file " + file;
  group.assign(n, 0u);
  uint32_t G = 0;
  for (uint32_t i = 0; i < n; i++) {
    unsigned int v = 0;
    in >> v;
    group[i] = v;
    G = std::max(G, v + 1);
  }
  return G;
}

// A relation block (block structure, BS) as the reference reads it for MCMC and ALS (relation.h:70-114): only its
// transposed matrix <stem>.xt, whose rows are the block's features and whose columns are its rows, and its optional
// <stem>.groups.  Every error names the file and starts with "relations: ".
struct RelationData {
  uint32_t num_cases = 0, num_feature = 0;
  uint32_t attr_offset = 0;  // model id of feature 0, set after the main table's attributes (libfm.cpp:213-216)
  std::vector<uint64_t> col_ptr{0};  // the .xt: feature j's entries at [col_ptr[j], col_ptr[j + 1])
  std::vector<uint32_t> row;
  std::vector<float> val;
  std::vector<uint32_t> attr_group;  // [num_feature]: its DataMetaInfo, all 0 without a .groups file
  uint32_t num_groups = 1;

  void load(const std::string& stem) {
    std::cout << "has x = " << 0 << std::endl;
    std::cout << "has xt = " << 1 << std::endl;
    std::cout << "data transpose... ";
    try {
      const SparseData::XHeader fh = SparseData::read_matrix(stem + ".xt", "", 0, true, col_ptr, row, val);
      num_feature = fh.num_rows;
      num_cases = fh.num_cols;
      std::cout << "num_cases=" << num_cases << "\tnum_values=" << fh.num_values << "\tnum_features=" << num_feature
                << std::endl;
      attr_group.assign(num_feature, 0u);
      num_groups = 1;
      if (SparseData::file_exists(stem + ".groups")) num_groups = read_groups(stem + ".groups", num_feature, attr_group);
    } catch (const std::string& e) {
      throw "relations: " + e;
    }
  }
};

// RelationJoin::load (relation.h:127-150): a data set's case -> block row map, binary when the file starts with a
// DVector<uint> header {1, 4}, else expected_rows whitespace-separated numbers.  Its length must be the data set's
// case count.
struct RelationJoin {
  std::vector<uint32_t> rows;

  void load(const std::string& file, uint64_t expected_rows) {
    std::ifstream in(file.c_str(), std::ios::binary);
    if (!in.is_open()) throw "relations: could not open " + file;
    uint32_t hdr[3] = {0, 0, 0};
    in.read(reinterpret_cast<char*>(hdr), 2 * sizeof(uint32_t));
    const bool binary = in && hdr[0] == 1 && hdr[1] == sizeof(uint32_t);
    uint64_t n = 0;
    if (binary) {
      in.read(reinterpret_cast<char*>(hdr + 2), sizeof(uint32_t));
      if (!in) throw "relations: could not read " + file;
      n = hdr[2];
      if (n == expected_rows) {
        rows.resize(n);
        in.read(reinterpret_cast<char*>(rows.data()), sizeof(uint32_t) * n);
        if (!in) throw "relations: could not read " + file;
      }
    } else {
      in.clear();
      in.close();
      std::ifstream txt(file.c_str());
      rows.clear();
      rows.reserve(expected_rows);
      unsigned int v;
      while (rows.size() < expected_rows && txt >> v) rows.push_back(v);
      n = rows.size();
    }
    if (n != expected_rows)
      throw "relations: " + file + " maps " + std::to_string(n) + " cases, its data set has " +
          std::to_string(expected_rows);
  }
};

// A binary data set read through a budget of host memory (-cache_size), in blocks of consecutive rows in
// file order, as the reference's LargeSparseMatrixHD (util/fmatrix.h:165-262) reads it through its row
// cache.  Only the targets are held whole.  The plan is greedy: a block takes rows while its .x bytes
// stay within cache_size / 2, so that two blocks fit the budget -- one in use, the next being read.
// The same holds for the transposed file <file>.xt that MCMC and ALS read (open_xt): its rows are the
// features (the columns of the data) and its ids the cases.
struct BinaryBlocks {
  struct Block {
    uint64_t row_lo = 0, row_hi = 0;  // rows [row_lo, row_hi)
    uint64_t nnz = 0;
    uint64_t offset = 0;  // file offset of row_lo's header
    uint64_t rows() const { return row_hi - row_lo; }
    uint64_t bytes() const { return 4 * rows() + 8 * nnz; }
  };
  std::string fx;
  bool transposed = false;  // fx is the .xt: rows are features, ids are cases
  uint64_t n_file_rows = 0;
  std::vector<float> target;
  float min_target = +std::numeric_limits<float>::max();
  float max_target = -std::numeric_limits<float>::max();
  int num_feature = 0;
  uint64_t num_values = 0;
  uint64_t budget = 0;  // .x bytes per block
  std::vector<Block> blocks;
  uint64_t max_block_rows = 0, max_block_bytes = 0;

  uint64_t num_cases() const { return target.size(); }

  // Null when `filename` is text input or its rows fit in one block: such a data set is loaded whole.
  static std::unique_ptr<BinaryBlocks> open(const std::string& filename, uint64_t cache_size) {
    std::string fx, fy;
    if (!SparseData::binary_pair(filename, &fx, &fy)) return nullptr;
    std::unique_ptr<BinaryBlocks> d(new BinaryBlocks());
    d->fx = fx;
    d->budget = cache_size / 2;
    d->target = SparseData::read_targets(fy);
    std::ifstream in(fx.c_str(), std::ios::binary);
    const SparseData::XHeader fh = SparseData::read_header(in, fx, fy, d->target.size());
    if (4ull * fh.num_rows + 8ull * fh.num_values <= d->budget) return nullptr;
    in.close();
    d->num_feature = (int)fh.num_cols;
    d->finish_open(fh);
    return d;
  }

  // The transposed file of `filename` (<file>.xt beside .x/.y, <file>.datat beside .data/.target; Data.h:124-152)
  // under the same budget.  Null when there is none, or its columns fit in one block: the data set is then
  // loaded whole, from .x.  num_feature is the .xt's row count (Data.h:157); its case count must match .y.
  static std::unique_ptr<BinaryBlocks> open_xt(const std::string& filename, uint64_t cache_size) {
    std::string fx, fy;
    if (!SparseData::binary_pair(filename, &fx, &fy) || !SparseData::file_exists(fx + "t")) return nullptr;
    std::unique_ptr<BinaryBlocks> d(new BinaryBlocks());
    d->fx = fx + "t";
    d->transposed = true;
    d->budget = cache_size / 2;
    d->target = SparseData::read_targets(fy);
    std::ifstream in(d->fx.c_str(), std::ios::binary);
    const SparseData::XHeader fh = SparseData::read_header(in, d->fx, fy, d->target.size(), true);
    if (4ull * fh.num_rows + 8ull * fh.num_values <= d->budget) return nullptr;
    in.close();
    d->num_feature = (int)fh.num_rows;
    d->finish_open(fh);
    return d;
  }

  // What Data::load prints for the file read (Data.h:113-176), and the plan
  void print() const {
    std::cout << "has x = " << !transposed << std::endl;
    std::cout << "has xt = " << transposed << std::endl;
    std::cout << (transposed ? "data transpose... " : "data... ") << "num_cases=" << num_cases()
              << "\tnum_values=" << num_values << "\tnum_features=" << num_feature << "\tmin_target=" << min_target
              << "\tmax_target=" << max_target << std::endl;
    std::cout << "streaming " << fx << ": " << blocks.size() << " blocks of at most " << max_block_rows
              << (transposed ? " columns and " : " rows and ") << budget << " bytes" << std::endl;
  }

  void binarize_targets() {  // libfm.cpp:302-303
    for (auto& t : target) t = (t <= 0.0f) ? -1.0f : 1.0f;
  }

 private:
  void finish_open(const SparseData::XHeader& fh) {
    n_file_rows = fh.num_rows;
    num_values = fh.num_values;
    for (float y : target) {  // Data.h:166-171
      if (y < min_target) min_target = y;
      if (y > max_target) max_target = y;
    }
    plan();
  }

  // Walk the row headers once (reading the file in large pieces, skipping rows that span one) and cut the
  // blocks.  The row count is the header's (for a .x already checked against the targets).
  void plan() {
    FILE* f = fopen(fx.c_str(), "rb");
    if (!f) throw "could not open " + fx;
    std::unique_ptr<FILE, int (*)(FILE*)> closer(f, fclose);
    fseeko(f, 0, SEEK_END);
    const uint64_t fsize = (uint64_t)ftello(f);
    std::vector<char> buf(16u << 20);
    uint64_t buf_lo = 0, buf_n = 0;  // file bytes [buf_lo, buf_lo + buf_n) are in buf
    uint64_t pos = sizeof(SparseData::XHeader), nnz = 0;
    Block cur;
    cur.offset = pos;
    for (uint64_t r = 0; r < n_file_rows; r++) {
      if (pos < buf_lo || pos + 4 > buf_lo + buf_n) {
        buf_lo = pos;
        buf_n = 0;
        if (fseeko(f, (off_t)pos, SEEK_SET) == 0) buf_n = fread(buf.data(), 1, buf.size(), f);
        if (buf_n < 4) throw "could not read " + fx;
      }
      uint32_t size;
      memcpy(&size, buf.data() + (pos - buf_lo), 4);
      const uint64_t bytes = 4 + 8ull * size;
      if (pos + bytes > fsize || nnz + size > num_values) {
        if (transposed)
          throw "column " + std::to_string(r) + " of " + fx + ": its header word " + std::to_string(size) +
              " runs past the file's " + std::to_string(num_values) + " entries";
        throw "could not read " + fx;
      }
      if (bytes > budget)
        throw (transposed ? "column " : "row ") + std::to_string(r) + " of " + fx + " takes " + std::to_string(bytes) +
            " bytes: -cache_size must be at least " + std::to_string(2 * bytes);
      if (cur.bytes() + bytes > budget) {
        add(cur);
        cur = Block();
        cur.row_lo = r;
        cur.offset = pos;
      }
      cur.row_hi = r + 1;
      cur.nnz += size;
      pos += bytes;
      nnz += size;
    }
    if (nnz != num_values) throw "could not read " + fx;
    if (cur.rows() > 0 || blocks.empty()) add(cur);
  }

  void add(const Block& b) {
    blocks.push_back(b);
    if (b.rows() > max_block_rows) max_block_rows = b.rows();
    if (b.bytes() > max_block_bytes) max_block_bytes = b.bytes();
  }
};

// One pass over a BinaryBlocks in file order.  A thread reads block b into buffer b % 2 -- its .x bytes
// as the file stores them, the rows' sizes from their headers, and their targets -- as soon as the user
// has released block b - 2, so that block b + 1 is read while block b is in use.  The buffers come from
// `alloc` (page-locked memory for the GPU's copy engine in the command line, plain memory in tests).
class BlockReader {
 public:
  struct Buffer {
    const char* x = nullptr;
    const uint32_t* row_size = nullptr;
    const float* target = nullptr;
  };
  using Alloc = std::function<void*(uint64_t)>;
  using Free = std::function<void(void*)>;

  BlockReader(const BinaryBlocks& d, const Alloc& alloc, Free release) : d_(d), free_(std::move(release)) {
    const uint64_t x_bytes = (d.max_block_bytes + 15) & ~15ull;
    for (int i = 0; i < 2; i++) {
      raw_[i] = static_cast<char*>(alloc(x_bytes + 8 * d.max_block_rows));
      rs_[i] = reinterpret_cast<uint32_t*>(raw_[i] + x_bytes);
      tg_[i] = reinterpret_cast<float*>(raw_[i] + x_bytes + 4 * d.max_block_rows);
    }
  }
  BlockReader(const BlockReader&) = delete;
  BlockReader& operator=(const BlockReader&) = delete;
  ~BlockReader() {
    stop();
    for (char* p : raw_)
      if (p) free_(p);
  }

  void start() {
    stop();
    read_ = released_ = 0;
    abort_ = false;
    error_.clear();
    thread_ = std::thread([this] { run(); });
  }

  // Block b, once read; throws what the reader met on the way to it.
  Buffer wait(size_t b) {
    std::unique_lock<std::mutex> lk(m_);
    cv_.wait(lk, [&] { return read_ > b || !error_.empty(); });
    if (read_ <= b) throw error_;
    return Buffer{raw_[b % 2], rs_[b % 2], tg_[b % 2]};
  }

  // Block b's buffer may be refilled (blocks are released in order).
  void release(size_t b) {
    {
      std::lock_guard<std::mutex> lk(m_);
      released_ = b + 1;
    }
    cv_.notify_all();
  }

  void stop() {
    {
      std::lock_guard<std::mutex> lk(m_);
      abort_ = true;
    }
    cv_.notify_all();
    if (thread_.joinable()) thread_.join();
  }

 private:
  void run() {
    FILE* f = fopen(d_.fx.c_str(), "rb");
    try {
      if (!f) throw "could not open " + d_.fx;
      for (size_t b = 0; b < d_.blocks.size(); b++) {
        {
          std::unique_lock<std::mutex> lk(m_);
          cv_.wait(lk, [&] { return abort_ || b < released_ + 2; });
          if (abort_) break;
        }
        read_block(f, d_.blocks[b], b % 2);
        {
          std::lock_guard<std::mutex> lk(m_);
          read_ = b + 1;
        }
        cv_.notify_all();
      }
    } catch (const std::string& e) {
      std::lock_guard<std::mutex> lk(m_);
      error_ = e;
    }
    if (f) fclose(f);
    cv_.notify_all();
  }

  // The rows' sizes come from the headers just read; they must still add up to the plan's.
  void read_block(FILE* f, const BinaryBlocks::Block& bl, int i) {
    const uint64_t bytes = bl.bytes();
    if (fseeko(f, (off_t)bl.offset, SEEK_SET) != 0 || fread(raw_[i], 1, bytes, f) != bytes)
      throw "could not read " + d_.fx;
    uint64_t pos = 0, nnz = 0;
    for (uint64_t r = 0; r < bl.rows(); r++) {
      if (pos + 4 > bytes) throw "could not read " + d_.fx;
      uint32_t size;
      memcpy(&size, raw_[i] + pos, 4);
      rs_[i][r] = size;
      pos += 4 + 8ull * size;
      nnz += size;
    }
    if (pos != bytes || nnz != bl.nnz) throw "could not read " + d_.fx;
    if (!d_.transposed) memcpy(tg_[i], d_.target.data() + bl.row_lo, 4 * bl.rows());
  }

  const BinaryBlocks& d_;
  Free free_;
  char* raw_[2] = {nullptr, nullptr};
  uint32_t* rs_[2] = {nullptr, nullptr};
  float* tg_[2] = {nullptr, nullptr};
  std::thread thread_;
  std::mutex m_;
  std::condition_variable cv_;
  size_t read_ = 0, released_ = 0;
  bool abort_ = false;
  std::string error_;
};

}  // namespace host
