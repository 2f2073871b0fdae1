"""CPU: host-side logic -- loaders, model init/IO, sharding, gloo all-reduce."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, digest
from libfm_b200 import Data, FmError, FmModel, synth
from libfm_b200 import dist as fdist

TRICKY = """# a comment line
5 0:1 7:0.5

   3.5\t2:1e-1   9:2   # trailing comment
-1
+2 4:-3.25 4:1
0 11:0
"""


@pytest.fixture()
def tricky_file(tmp_path):
    p = tmp_path / "tricky.libfm"
    p.write_text(TRICKY)
    return str(p)


def test_python_loader_matches_reference_loader(tricky_file, ref_golden):
    g = ref_golden
    d = Data.load(tricky_file)
    assert np.array_equal(d.row_ptr, g["tricky_row_ptr"]) and np.array_equal(d.col, g["tricky_col"])
    assert np.array_equal(d.val, g["tricky_val"]) and np.array_equal(d.target, g["tricky_target"])
    assert [d.num_feature, d.min_target, d.max_target] == g["tricky_meta"].tolist()


def test_python_loader_rejects_garbage(tmp_path):
    p = tmp_path / "bad.libfm"
    p.write_text("1 3:1 oops\n")
    with pytest.raises(FmError, match="cannot parse line"):
        Data.load(str(p))
    with pytest.raises(FmError, match="unable to open"):
        Data.load(str(tmp_path / "missing"))


def test_model_init_draw_order_bit_exact(ref_golden):
    fm = FmModel(37, 5)
    fm.init_stdev = 0.1
    fm.init(seed=42)
    g = ref_golden
    assert fm.w0 == g["init37_w0"] and np.array_equal(fm.w, g["init37_w"]) and np.array_equal(fm.v, g["init37_v"])


def checkpoint_model():
    fm = FmModel(12, 3)
    fm.init_stdev = 0.1
    fm.init(seed=3)
    fm.w0, fm.w[:] = 0.125, np.linspace(-1, 1, 12)
    return fm


def test_model_text_checkpoint_readable_by_reference(tmp_path, ref_golden):
    """The reference's fm_model::loadModel of this checkpoint, and its saveModel afterwards (stored)."""
    fm = checkpoint_model()
    path = str(tmp_path / "m.txt")
    fm.saveModel(path)
    g = ref_golden
    g6 = lambda a: np.array([float("%g" % x) for x in np.ravel(a)]).reshape(np.shape(a))  # noqa: E731
    assert g["ckpt_w0"] == 0.125 and np.array_equal(g["ckpt_w"], g6(fm.w)) and np.array_equal(g["ckpt_v"], g6(fm.v))
    assert str(g["ckpt_text"]) == open(path).read()  # idempotent text form


def cli_loader_args(path):
    return ["-task", "r", "-train", path, "-test", path, "-method", "sgd", "-iter", "0", "-learn_rate", "0.01",
            "-seed", "1"]


def loader_lines(stdout):
    return [l for l in stdout.splitlines() if l.startswith("num_rows=") or l.startswith("has x")]


def test_cli_loader_lines_match_reference(tricky_file, tmp_path, ref_golden):
    """bin/libFM parses its inputs before it needs a GPU: its loader summary lines must
    equal the reference CLI's, byte for byte."""
    cli = os.path.join(ROOT, "bin", "libFM")
    if not os.path.exists(cli):
        pytest.skip("CLI binaries not built")
    ours = subprocess.run([cli] + cli_loader_args(tricky_file), capture_output=True, text=True)
    want = ref_golden["cli_loader_lines"].tolist()
    assert loader_lines(ours.stdout) == want and len(want) == 6
    import torch
    if not torch.cuda.is_available():
        assert ours.returncode != 0 and "no CPU path" in ours.stderr


def test_reference_main_links_against_the_c_abi(tricky_file):
    """integration/fm_learn_sgd_b200.h compiled into the reference's own main() (oracle/_ref/libFM_b200):
    the C ABI binds to the reference's Data / DVector / sparse_row types, the binary resolves
    libfmb200.so through its rpath, and without a GPU it refuses loudly instead of training on the CPU."""
    from oracle.binding import REF_CLI_B200
    if not os.path.exists(REF_CLI_B200):
        pytest.skip("oracle/_ref/libFM_b200 not built (no /root/reference here)")
    args = ["-task", "r", "-train", tricky_file, "-test", tricky_file, "-method", "sgd",
            "-iter", "1", "-learn_rate", "0.01", "-seed", "1"]
    r = subprocess.run([REF_CLI_B200] + args, capture_output=True, text=True)
    assert "num_rows=" in r.stdout  # the reference's loader ran
    import torch
    if not torch.cuda.is_available():
        assert "no CPU path" in r.stderr and "#Iter" not in r.stdout


def test_cli_flag_errors_match_reference_text(tmp_path):
    cli = os.path.join(ROOT, "bin", "libFM")
    if not os.path.exists(cli):
        pytest.skip("CLI not built")
    r = subprocess.run([cli, "-task", "r", "-bogus", "1"], capture_output=True, text=True)
    assert "ERROR: the parameter bogus does not exist" in r.stderr
    r = subprocess.run([cli, "-task", "r", "-task", "c"], capture_output=True, text=True)
    assert "ERROR: the parameter task is already specified" in r.stderr
    r = subprocess.run([cli, "-task", "r", "-train", "x", "-test", "y"], capture_output=True, text=True)
    assert "outside the libfm_b200 scope" in r.stderr  # default method is mcmc (libfm.cpp:118)


def test_shard_bounds_partition_rows():
    for n in (0, 1, 7, 1000, 1_000_209):
        for world in (1, 2, 3, 8):
            b = [fdist.shard_bounds(n, world, r) for r in range(world)]
            assert b[0][0] == 0 and b[-1][1] == n
            assert all(b[i][1] == b[i + 1][0] for i in range(world - 1))
            sizes = [hi - lo for lo, hi in b]
            assert max(sizes) - min(sizes) <= 1
    d = synth.ragged(101, 30, 5, seed=1)
    parts = [fdist.shard(d, 4, r) for r in range(4)]
    assert sum(p.num_cases for p in parts) == d.num_cases
    assert np.array_equal(np.concatenate([p.col for p in parts]), d.col)
    assert np.array_equal(np.concatenate([p.target for p in parts]), d.target)
    assert all(p.row_ptr[0] == 0 for p in parts)


_WORKER = r"""
import os, sys, json
sys.path.insert(0, %(root)r)
import torch, torch.distributed as dist
from libfm_b200 import dist as fdist, synth
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%(port)d", rank=int(sys.argv[1]), world_size=2)
world, rank = 2, int(sys.argv[1])
# each rank holds a different replica; after the epoch's all-reduce both hold the mean
p = torch.arange(10, dtype=torch.float32) * (rank + 1)
fdist.allreduce_mean_(p, world)
assert torch.allclose(p, torch.arange(10, dtype=torch.float32) * 1.5), p
d = synth.ragged(101, 30, 5, seed=1)
mine = fdist.shard(d, world, rank)
sq, ab, ok, n = fdist.sum_metrics(float(mine.num_cases), 2.0, mine.num_cases, mine.num_cases, world)
assert n == d.num_cases and ok == d.num_cases and sq == float(d.num_cases) and ab == 4.0
# the mean-field exchange (same rule as fm_peer_meanfield_kernel): two replicas that moved away from a common
# theta0 on their own shards combine to theta0 + gamma_i * (delta_0 + delta_1); both ranks end identical and
# equal to a numpy restatement computed from the same seeds
import numpy as np
n_f, kp, ws = 12, 4, 8
off_w, off_v = 4, 4 + n_f * ws
size = off_v + n_f * kp
g0 = np.random.default_rng(5)
theta0 = torch.tensor(g0.standard_normal(size).astype(np.float32) * 0.1)
deltas = [np.random.default_rng(10 + r).standard_normal(size).astype(np.float32) * 0.01 for r in range(2)]
counts = [np.random.default_rng(20 + r).integers(0, 400, n_f).astype(np.float32) for r in range(2)]
rows = [1000, 1200]
mine_p = theta0 + torch.tensor(deltas[rank])
lay = dict(off_w=off_w, ws=ws, off_v=off_v, kp=kp, n=n_f)
fdist.combine_meanfield_(mine_p, theta0, torch.tensor(counts[rank]), rows[rank], lay, lr=0.01, regw=0.001, regv=0.002, world=2)
def gam(u, G=2.0):
    u = np.asarray(u, dtype=np.float64); out = np.ones_like(u); m = u > 1e-6
    out[m] = -np.expm1(-G * u[m]) / (G * -np.expm1(-u[m])); return out
t0 = theta0.numpy().astype(np.float64)
cm = (counts[0] + counts[1]) / 2.0
hv = float((t0[off_v:] ** 2).sum()) / n_f
gamma = np.zeros(size)
gamma[0] = gam(np.array([0.01 * np.mean(rows)]))[0]
gamma[off_w:off_v:ws] = gam(0.01 * 1.001 * cm)
gamma[off_v:] = np.repeat(gam(0.01 * (hv + 0.002) * cm), kp)
want = t0 + gamma * (deltas[0].astype(np.float64) + deltas[1].astype(np.float64))
assert np.allclose(mine_p.numpy(), want, atol=2e-6), np.abs(mine_p.numpy() - want).max()
both = [torch.zeros_like(mine_p) for _ in range(2)]
dist.all_gather(both, mine_p)
assert torch.equal(both[0], both[1])
dist.destroy_process_group()
print("rank", rank, "ok")
"""


def test_world_size_2_gloo_allreduce_and_shards(tmp_path):
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    script = tmp_path / "w.py"
    script.write_text(_WORKER % {"root": ROOT, "port": port})
    procs = [subprocess.Popen([sys.executable, str(script), str(r)], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=120)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs


def test_product_never_touches_the_oracle():
    """oracle/ is test infrastructure: nothing under libfm_b200/ (Python, C++, CUDA) may
    import, include, link or dlopen it."""
    import re
    bad = []
    for root, _, files in os.walk(os.path.join(ROOT, "libfm_b200")):
        if "__pycache__" in root:
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(root, f), errors="ignore").read()
                if re.search(r"(import\s+oracle|from\s+oracle|libfm_oracle|libfm_ref|oracle/)", txt):
                    bad.append(os.path.join(root, f))
    assert not bad, bad


def test_bench_reference_arm_line(tmp_path):
    """`bench.py --impl reference` runs the reference's CPU row loop and prints the contract's JSON."""
    import json
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "2",
                        "--warmup", "1"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["unit"] == "examples/s" and line["higher_is_better"] is True
    assert line["metric"].startswith("MovieLens-1M-shaped examples/sec")
    assert line["cpu_baseline"]["cores"] == 1 and line["cpu_baseline"]["kind"] in ("reference", "port")
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["e2e"]["value"] == line["value"]
    assert 1e6 < line["value"] < 1e9  # a single CPU core: tens of millions of examples/s


@pytest.fixture(scope="module")
def loader_dump(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("bin") / "loader_dump")
    subprocess.run(["g++", "-O2", "-std=c++17", "-pthread", "-I", os.path.join(ROOT, "libfm_b200", "host"),
                    os.path.join(ROOT, "tests", "loader_dump.cpp"), "-o", exe], check=True)
    return exe


def _read_dump(path):
    raw = open(path, "rb").read()
    n, nnz, nf = np.frombuffer(raw, np.uint64, 2, 0).tolist() + [int(np.frombuffer(raw, np.int64, 1, 16)[0])]
    mn, mx = np.frombuffer(raw, np.float32, 2, 24)
    o = 32
    rp = np.frombuffer(raw, np.uint64, n + 1, o); o += 8 * (n + 1)
    col = np.frombuffer(raw, np.uint32, nnz, o); o += 4 * nnz
    val = np.frombuffer(raw, np.float32, nnz, o); o += 4 * nnz
    tgt = np.frombuffer(raw, np.float32, n, o)
    return rp, col, val, tgt, nf, float(mn), float(mx)


def _file_digest(path):
    return digest(np.frombuffer(open(path, "rb").read(), np.uint8))


def _csr_digest(csr):
    return "".join(digest(a) for a in csr[:4])


def write_threaded_input(path):
    r = np.random.default_rng(5)
    with open(path, "w") as f:
        f.write("# header comment\n\n")
        for i in range(60_000):
            z = int(r.integers(0, 7))
            ids = r.integers(0, 5000, z)
            vals = r.standard_normal(z)
            lead = "  " if i % 97 == 0 else ""
            tail = "   # c" if i % 53 == 0 else ("\t" if i % 31 == 0 else "")
            f.write(lead + "%g" % r.integers(-3, 6) + "".join(" %d:%.6g" % (a, b) for a, b in zip(ids, vals)) + tail + "\n")
            if i % 1000 == 0:
                f.write("\n# interleaved comment\n")
        f.write("4 7:1")  # last line without a newline


def test_cli_loader_threaded_text_equals_reference(loader_dump, tmp_path, ref_golden):
    """A > 1 MB text file takes the multi-threaded path of host/sparse_data.h (cut at
    line boundaries, parsed by all cores, concatenated in file order): the CSR must be
    bit-identical to what the reference's two-pass sscanf loader builds."""
    path = str(tmp_path / "big.libfm")
    write_threaded_input(path)
    assert os.path.getsize(path) > (1 << 20)
    assert _file_digest(path) == ref_golden["threaded_input_sha"]  # the input the reference read
    out = str(tmp_path / "dump.bin")
    subprocess.run([loader_dump, path, out], check=True)
    got = _read_dump(out)
    assert _csr_digest(got) == ref_golden["threaded_csr_sha"]
    assert list(got[4:]) == ref_golden["threaded_meta"].tolist()


def test_cli_loader_reports_first_error_in_file_order(loader_dump, tmp_path):
    path = str(tmp_path / "bad.libfm")
    with open(path, "w") as f:
        for i in range(120_000):
            f.write("1 3:1 4:2\n" if i not in (70_000, 110_000) else "1 3:1 oops%d\n" % i)
    r = subprocess.run([loader_dump, path, str(tmp_path / "x.bin")], capture_output=True, text=True)
    assert r.returncode == 1 and 'cannot parse line "1 3:1 oops70000" at character o' in r.stderr


def write_convert_input(path):
    synth.to_libfm_text(synth.ragged(80_000, 3000, 6, seed=4), path)


def test_convert_tool_output_is_byte_identical_to_reference(tricky_file, tmp_path, ref_golden):
    """bin/convert (host/convert_main.cpp) vs the reference's convert tool: same flags,
    byte-identical .x / .y files -- also on a file large enough for the threaded parser."""
    ours = os.path.join(ROOT, "bin", "convert")
    if not os.path.exists(ours):
        pytest.skip("convert binaries not built")
    big = str(tmp_path / "big.libfm")
    write_convert_input(big)
    assert os.path.getsize(big) > (1 << 20)
    assert _file_digest(big) == ref_golden["convert_big_input_sha"]
    for tag, src in (("tricky", tricky_file), ("big", big)):
        x, y = str(tmp_path / "a.x"), str(tmp_path / "a.y")
        r = subprocess.run([ours, "--ifile", src, "--ofilex", x, "--ofiley", y], capture_output=True, text=True)
        assert os.path.exists(x), r.stderr
        assert _file_digest(x) + _file_digest(y) == ref_golden["convert_%s_sha" % tag]


def fuzz_inputs():
    """40 randomised libfm texts (odd spacing, signs, exponents, comments, blank lines, empty rows,
    every fourth with a garbage line)."""
    r = np.random.default_rng(2024)

    def num(x):
        return r.choice(["%g", "%.3f", "%e", "%+g"]) % x

    def line():
        kind = r.random()
        if kind < 0.05:
            return r.choice(["", "   ", "\t", "# only a comment", "  # indented comment"])
        y = num(r.normal() * 3)
        ents = " ".join("%s%d:%s" % ("" if r.random() < 0.8 else " ", int(r.integers(0, 300)), num(r.normal()))
                        for _ in range(int(r.integers(0, 6))))
        s = r.choice(["", " ", "\t"]) + y + (" " + ents if ents else "") + r.choice(["", " ", "  # tail", "\t\t"])
        return s

    bad_tails = ["1 3:1 x", "abc", "1 3 :1", "2 4:", "1 5:1 6", "3 7:1e", "1 2:3:4"]
    for trial in range(40):
        lines = [line() for _ in range(int(r.integers(1, 60)))]
        if trial % 4 == 3:
            lines.insert(int(r.integers(0, len(lines) + 1)), str(r.choice(bad_tails)))
        yield "\n".join(lines) + ("\n" if r.random() < 0.7 else "")


def test_cli_loader_fuzz_against_reference(loader_dump, tmp_path, ref_golden):
    """Randomised libfm text through host/sparse_data.h, against what the reference's Data::load
    made of the same texts: identical CSR, or the same `cannot parse line` error."""
    g = ref_golden
    for trial, text in enumerate(fuzz_inputs()):
        path = str(tmp_path / ("f%d.libfm" % trial))
        with open(path, "w") as f:
            f.write(text)
        assert _file_digest(path) == g["fuzz_input_sha"][trial], trial  # the text the reference read
        out = str(tmp_path / "d.bin")
        ours = subprocess.run([loader_dump, path, out], capture_output=True, text=True)
        err = str(g["fuzz_error"][trial])
        if err:
            assert ours.returncode == 1, (trial, text, err)
            assert err in ours.stderr, (err, ours.stderr)
            continue
        assert ours.returncode == 0, (trial, ours.stderr, text)
        got = _read_dump(out)
        assert _csr_digest(got) == g["fuzz_csr_sha"][trial], (trial, text)
        assert list(got[4:]) == g["fuzz_meta"][trial].tolist(), (trial, got[4:])
