// wavefront_host.cpp -- TEST INFRASTRUCTURE.  Compiles the wavefront kernels' own source
// (libfm_b200/csrc/fm_inorder_wavefront.cuh, fm_sgda_wavefront.cuh) for the host through
// simt_shim.h, runs each as 32 threads on seeded synthetic data and compares the resulting state
// bit for bit with the sequential oracle: w0 / w / V with fmo_sgd_epoch (oracle/fm_oracle.c), and
// w0 / w / V / grad_w / grad_v / reg_w / reg_v with fmo_sgda_epoch (oracle/fm_oracle_sgda.c).
// Exit status 0 = every case identical.
// Built twice by tests/test_simt_wavefront.py: plain, and with -fsanitize=thread.
#include "simt_shim.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

#include "../../libfm_b200/csrc/fm_inorder_wavefront.cuh"
#include "../../libfm_b200/csrc/fm_sgda_wavefront.cuh"

namespace simt {
thread_local Dim tid;
pthread_barrier_t warp_barrier;
unsigned ballot_in[kLanes];
uint64_t shfl_in[kLanes];
alignas(16) double dynamic_smem[4096];
}  // namespace simt

extern "C" void fmo_sgd_epoch(uint32_t n, int k, int k0, int k1, double* w0, double* w, double* v, double lr,
                              double reg0, double regw, double regv, int task, double min_target,
                              double max_target, uint64_t n_rows, const uint64_t* row_ptr,
                              const uint32_t* col, const float* val, const float* target);
extern "C" void fmo_sgda_epoch(uint32_t n, int k, int k0, int k1, double* w0, double* w, double* v, double* grad_w,
                               double* grad_v, double* reg_w, double* reg_v, const uint32_t* group, uint32_t n_groups,
                               double lr, int task, double min_target, double max_target, int lambda_steps,
                               uint64_t n_rows, const uint64_t* row_ptr, const uint32_t* col, const float* val,
                               const float* target, uint64_t v_rows, const uint64_t* v_row_ptr, const uint32_t* v_col,
                               const float* v_val, const float* v_target);

namespace {

struct Rng {  // xorshift64*
  uint64_t s;
  explicit Rng(uint64_t seed) : s(seed * 0x9E3779B97F4A7C15ull + 1) {}
  uint64_t next() {
    s ^= s >> 12;
    s ^= s << 25;
    s ^= s >> 27;
    return s * 0x2545F4914F6CDD1Dull;
  }
  double uni() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
  uint32_t below(uint32_t n) { return (uint32_t)(uni() * n); }
  double gauss() {  // sum of uniforms: shape is irrelevant here
    double a = 0;
    for (int i = 0; i < 6; i++) a += uni();
    return (a - 3.0) * 1.41;
  }
};

struct Case {
  const char* name;
  uint64_t n_rows;
  uint32_t n_feat;
  int k, k0, k1, task;
  double regs[3];
  double skew;     // ids ~ n * u^skew (1 = uniform; larger = a few hot features)
  bool ragged;     // 0..4 entries with real values, else exactly 2 one-hot entries
  int dup_every;   // every so many rows repeat the first id inside the row
};

struct Csr {
  std::vector<uint64_t> row_ptr;
  std::vector<uint32_t> col;
  std::vector<float> val, target;
};

Csr make_data(const Case& c, uint64_t seed) {
  Rng r(seed);
  Csr d;
  d.row_ptr.push_back(0);
  auto draw = [&](uint32_t lo, uint32_t span) {
    double u = r.uni();
    double t = 1.0;
    for (int i = 0; i < (int)c.skew; i++) t *= u;
    return lo + (uint32_t)(t * span) % span;
  };
  for (uint64_t i = 0; i < c.n_rows; i++) {
    int size = c.ragged ? (int)r.below(5) : 2;
    for (int j = 0; j < size; j++) {
      if (c.ragged) {
        d.col.push_back(draw(0, c.n_feat));
        d.val.push_back((float)(r.gauss() * 0.7));
      } else {
        uint32_t half = c.n_feat / 2;
        d.col.push_back(j == 0 ? draw(0, half) : draw(half, c.n_feat - half));
        d.val.push_back(1.0f);
      }
    }
    if (c.dup_every && i % c.dup_every == 0 && size >= 2) d.col.back() = d.col[d.col.size() - size];
    d.row_ptr.push_back(d.col.size());
    float y = (float)(1 + r.below(5));
    if (c.task == 1) y = y > 3 ? 1.0f : -1.0f;
    d.target.push_back(y);
  }
  return d;
}

template <bool K0, int TASK>
void run_lanes(fmb::Params64 p, const Case& c, fmb::HParams hp, const Csr& d) {
  std::vector<std::thread> lanes;
  for (unsigned l = 0; l < simt::kLanes; l++)
    lanes.emplace_back([&, l] {
      simt::tid.x = l;
      fmb::fm_sgd_inorder_wavefront_kernel<K0, TASK>(p, c.k, c.k0, c.k1, hp, c.n_rows, d.row_ptr.data(),
                                                     d.col.data(), d.val.data(), d.target.data());
    });
  for (auto& t : lanes) t.join();
}

bool run_case(const Case& c, int epochs) {
  const Csr d = make_data(c, 1234);
  const uint32_t n = c.n_feat;
  const int k = c.k;
  Rng r(99);
  // oracle state: factor-major V [k][n]; device state: Params64 [w0, pad | w[n] (even) | V[n][k]]
  double w0 = 0.05;
  std::vector<double> w(n), v((size_t)k * n);
  for (auto& x : w) x = r.gauss() * 0.1;
  for (auto& x : v) x = r.gauss() * 0.1;
  const size_t OW = fmb::Params64::off_w, OV = OW + (((size_t)n + 1) & ~(size_t)1);
  std::vector<double> dev(OV + (size_t)n * k + 2);
  dev[0] = w0;
  for (uint32_t i = 0; i < n; i++) dev[OW + i] = w[i];
  for (int f = 0; f < k; f++)
    for (uint32_t i = 0; i < n; i++) dev[OV + (size_t)i * k + f] = v[(size_t)f * n + i];
  fmb::Params64 p;
  p.base = dev.data();
  p.n_doubles = dev.size();
  p.off_v = OV;
  fmb::HParams hp;
  hp.task = c.task;
  hp.lr = 0.02;
  hp.reg0 = c.regs[0];
  hp.regw = c.regs[1];
  hp.regv = c.regs[2];
  hp.min_target = c.task == 0 ? 1.0 : -1.0;
  hp.max_target = c.task == 0 ? 4.0 : 1.0;  // ratings reach 5: both clamp branches are exercised
  for (int e = 0; e < epochs; e++) {
    fmo_sgd_epoch(n, k, c.k0, c.k1, &w0, w.data(), v.data(), hp.lr, hp.reg0, hp.regw, hp.regv, hp.task,
                  hp.min_target, hp.max_target, c.n_rows, d.row_ptr.data(), d.col.data(), d.val.data(),
                  d.target.data());
    if (c.k0 && c.task == 0) run_lanes<true, 0>(p, c, hp, d);
    else if (c.k0) run_lanes<true, 1>(p, c, hp, d);
    else if (c.task == 0) run_lanes<false, 0>(p, c, hp, d);
    else run_lanes<false, 1>(p, c, hp, d);
  }
  uint64_t bad = 0;
  if (c.k0 && memcmp(&dev[0], &w0, 8) != 0) bad++;
  if (!c.k0 && dev[0] != 0.05) bad++;  // no bias: untouched
  for (uint32_t i = 0; i < n; i++)
    if (memcmp(&dev[OW + i], &w[i], 8) != 0) bad++;
  for (int f = 0; f < k; f++)
    for (uint32_t i = 0; i < n; i++)
      if (memcmp(&dev[OV + (size_t)i * k + f], &v[(size_t)f * n + i], 8) != 0) bad++;
  printf("%-16s rows=%llu n=%u k=%d  %s (%llu differing values)\n", c.name, (unsigned long long)c.n_rows, n, k,
         bad ? "MISMATCH" : "bit-identical", (unsigned long long)bad);
  return bad == 0;
}

// ---- SGDA ----------------------------------------------------------------------------------

struct SgdaCase {
  const char* name;
  uint64_t n_rows, v_rows;
  uint32_t n_feat, n_groups;
  int k, k0, k1, task;
  double skew;
  bool ragged;
  int dup_every;
  bool echo;  // validation row t repeats train row t (t % 3 == 0) or t + 1 (t % 3 == 1)
};

void run_sgda_lanes(const fmb::SgdaArgs& a) {
  std::vector<std::thread> lanes;
  for (unsigned l = 0; l < simt::kLanes; l++)
    lanes.emplace_back([&, l] {
      simt::tid.x = l;
      fmb::fm_sgda_wavefront_kernel(a);
    });
  for (auto& t : lanes) t.join();
}

bool run_sgda_case(const SgdaCase& c, int epochs) {
  const Case shape{c.name, c.n_rows, c.n_feat, c.k, c.k0, c.k1, c.task, {0, 0, 0}, c.skew, c.ragged, c.dup_every};
  const Csr d = make_data(shape, 1234);
  Case vshape = shape;
  vshape.n_rows = c.v_rows;
  Csr va = make_data(vshape, 4321);
  if (c.echo) {  // rebuild the validation rows, copying train rows where the case asks for it
    Csr e;
    e.row_ptr.push_back(0);
    for (uint64_t t = 0; t < c.v_rows; t++) {
      const bool copy = t % 3 < 2 && t + t % 3 < c.n_rows;
      const Csr& src = copy ? d : va;
      const uint64_t r = copy ? t + t % 3 : t;
      for (uint64_t i = src.row_ptr[r]; i < src.row_ptr[r + 1]; i++) {
        e.col.push_back(src.col[i]);
        e.val.push_back(src.val[i]);
      }
      e.row_ptr.push_back(e.col.size());
      e.target.push_back(va.target[t]);
    }
    va = e;
  }
  const uint32_t n = c.n_feat, G = c.n_groups;
  const int k = c.k;
  Rng r(77);
  std::vector<uint32_t> group(n);
  for (auto& g : group) g = r.below(G);
  // oracle state: factor-major V and grad_v [k][n]; device state: Params64, grad_v [n][k]
  double w0 = 0.05;
  std::vector<double> w(n), v((size_t)k * n), gw(n, 0.0), gv((size_t)k * n, 0.0), rw(G), rv((size_t)G * k);
  for (auto& x : w) x = r.gauss() * 0.1;
  for (auto& x : v) x = r.gauss() * 0.1;
  for (auto& x : rw) x = r.uni() * 0.05;
  for (auto& x : rv) x = r.uni() * 0.05;
  const size_t OW = fmb::Params64::off_w, OV = OW + (((size_t)n + 1) & ~(size_t)1);
  std::vector<double> dev(OV + (size_t)n * k + 2), dgw(n, 0.0), dgv((size_t)n * k, 0.0), drw = rw, drv = rv;
  dev[0] = w0;
  for (uint32_t i = 0; i < n; i++) dev[OW + i] = w[i];
  for (int f = 0; f < k; f++)
    for (uint32_t i = 0; i < n; i++) dev[OV + (size_t)i * k + f] = v[(size_t)f * n + i];
  fmb::SgdaArgs a{};
  a.p.base = dev.data();
  a.p.n_doubles = dev.size();
  a.p.off_v = OV;
  a.grad_w = dgw.data();
  a.grad_v = dgv.data();
  a.reg_w = drw.data();
  a.reg_v = drv.data();
  a.group = group.data();
  a.n_groups = G;
  a.k = k;
  a.use_w0 = c.k0;
  a.use_w = c.k1;
  a.hp.task = c.task;
  a.hp.lr = 0.02;
  a.hp.min_target = c.task == 0 ? 1.0 : -1.0;
  a.hp.max_target = c.task == 0 ? 4.0 : 1.0;  // ratings reach 5: both clamp branches are exercised
  a.n_rows = c.n_rows;
  a.v_rows = c.v_rows;
  a.row_ptr = d.row_ptr.data();
  a.col = d.col.data();
  a.val = d.val.data();
  a.target = d.target.data();
  a.v_row_ptr = va.row_ptr.data();
  a.v_col = va.col.data();
  a.v_val = va.val.data();
  a.v_target = va.target.data();
  for (int e = 0; e < epochs; e++) {
    a.lambda_steps = e > 0;  // the reference's first epoch has no lambda-steps
    fmo_sgda_epoch(n, k, c.k0, c.k1, &w0, w.data(), v.data(), gw.data(), gv.data(), rw.data(), rv.data(),
                   group.data(), G, a.hp.lr, c.task, a.hp.min_target, a.hp.max_target, a.lambda_steps, c.n_rows,
                   d.row_ptr.data(), d.col.data(), d.val.data(), d.target.data(), c.v_rows, va.row_ptr.data(),
                   va.col.data(), va.val.data(), va.target.data());
    // as launch_sgda_epoch: cut at theta-step t*, the second launch restarting from a full cursor
    const uint64_t t_star = fmb::sgda_last_moments_step(c.n_rows, c.v_rows, a.lambda_steps);
    const uint64_t cut = t_star ? 2 * t_star + 1 : 0;
    if (cut) {
      a.h_begin = 0, a.h_end = cut, a.vc0 = 0;
      run_sgda_lanes(a);
    }
    a.h_begin = cut, a.h_end = 2 * c.n_rows, a.vc0 = cut ? c.v_rows : 0;
    run_sgda_lanes(a);
  }
  uint64_t bad = 0;
  auto differ = [&](const double* x, const double* y) { bad += memcmp(x, y, 8) != 0; };
  differ(&dev[0], &w0);
  for (uint32_t i = 0; i < n; i++) {
    differ(&dev[OW + i], &w[i]);
    differ(&dgw[i], &gw[i]);
    for (int f = 0; f < k; f++) {
      differ(&dev[OV + (size_t)i * k + f], &v[(size_t)f * n + i]);
      differ(&dgv[(size_t)i * k + f], &gv[(size_t)f * n + i]);
    }
  }
  for (uint32_t g = 0; g < G; g++) differ(&drw[g], &rw[g]);
  for (size_t i = 0; i < rv.size(); i++) differ(&drv[i], &rv[i]);
  printf("sgda_%-16s rows=%llu val=%llu n=%u k=%d G=%u  %s (%llu differing values)\n", c.name,
         (unsigned long long)c.n_rows, (unsigned long long)c.v_rows, n, k, G, bad ? "MISMATCH" : "bit-identical",
         (unsigned long long)bad);
  return bad == 0;
}

}  // namespace

int main(int argc, char** argv) {
  const double scale = argc > 1 ? atof(argv[1]) : 1.0;  // TSan builds run a fraction of the rows
  // "sgd": the SGD cases only.  The SGDA kernel's __shfl_sync sits in branches on values the lanes
  // read from shared memory, so with its barriers compiled out the lanes can disagree on them and
  // the shuffles' barriers no longer pair up.
  const bool with_sgda = !(argc > 2 && strcmp(argv[2], "sgd") == 0);
  pthread_barrier_init(&simt::warp_barrier, nullptr, simt::kLanes);
  const Case cases[] = {
      {"tiny", 5, 6, 8, 1, 1, 0, {0, 0, 0}, 1, false, 0},
      {"c2_shape", 6000, 9746, 8, 1, 1, 0, {0, 0, 0}, 1, false, 0},
      {"skewed", 4000, 600, 8, 1, 1, 0, {0, 0, 0}, 3, false, 0},
      {"ragged", 4000, 500, 8, 1, 1, 0, {0, 0, 0}, 2, true, 0},
      {"dups", 4000, 300, 8, 1, 1, 0, {0, 0, 0}, 2, true, 7},
      {"classification", 3000, 800, 8, 1, 1, 1, {0, 0, 0}, 1, false, 0},
      {"no_bias_no_w", 3000, 800, 8, 0, 0, 0, {0, 0, 0}, 1, false, 0},
      {"k3_reg", 3000, 400, 3, 1, 1, 0, {0.01, 0.02, 0.03}, 2, true, 0},
      {"k0_model", 2000, 400, 0, 1, 1, 0, {0, 0.01, 0}, 1, false, 0},
  };
  bool ok = true;
  for (Case c : cases) {
    c.n_rows = (uint64_t)(c.n_rows * scale) > 5 ? (uint64_t)(c.n_rows * scale) : 5;
    ok = run_case(c, 2) && ok;
  }
  const SgdaCase sgda_cases[] = {
      // name, train rows, validation rows, features, groups, k, k0, k1, task, skew, ragged, dup_every, echo
      {"dense", 1500, 400, 40, 3, 8, 1, 1, 0, 2, true, 0, false},
      {"echo", 1500, 1500, 600, 1, 5, 1, 1, 0, 1, false, 0, true},
      {"short_cursor", 1500, 7, 300, 3, 8, 1, 1, 0, 1, true, 0, false},
      {"dups_x", 1500, 300, 200, 3, 5, 1, 1, 0, 2, true, 5, false},
      {"k1", 1500, 250, 300, 1, 1, 1, 1, 0, 1, true, 0, true},
      {"classification", 1200, 200, 400, 3, 8, 1, 1, 1, 1, false, 0, false},
      {"no_bias_no_w", 1200, 200, 400, 3, 5, 0, 0, 0, 2, true, 0, false},
  };
  for (SgdaCase c : sgda_cases) {
    if (!with_sgda) break;
    c.n_rows = (uint64_t)(c.n_rows * scale) > 5 ? (uint64_t)(c.n_rows * scale) : 5;
    c.v_rows = (uint64_t)(c.v_rows * scale) > 3 ? (uint64_t)(c.v_rows * scale) : 3;
    ok = run_sgda_case(c, 3) && ok;
  }
  return ok ? 0 : 1;
}
