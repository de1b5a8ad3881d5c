"""CPU tests of the host side: C-ABI library loads and exports the declared surface (no compute
calls), graph containers reproduce the reference reader, config keeps the reference's names."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tests.golden import loader

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cabi_library_exports_every_declared_symbol():
    from graphgan_b200 import _cabi
    header = open(os.path.join(ROOT, "include", "graphgan_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b(gg_[a-z0-9_]+)\s*\(", header))
    assert declared, "header parse failed"
    lib = _cabi.lib()                       # loads without a GPU; binds all of _cabi.SIGNATURES
    assert declared == set(_cabi.SIGNATURES), (declared ^ set(_cabi.SIGNATURES))
    for name in declared:
        assert hasattr(lib, name)
    assert lib.gg_abi_version() == _cabi.ABI_VERSION
    # struct layout agreed between ctypes and the header (field count and a few offsets)
    fields = [f[0] for f in _cabi.WalkDesc._fields_]
    struct_src = header[header.index("typedef struct gg_walk_desc"):header.index("} gg_walk_desc;")]
    in_header = re.findall(r"[\w\s\*]+?\b(\w+);", struct_src)
    assert fields == [f for f in in_header if f != "gg_walk_desc"]
    assert C.sizeof(_cabi.WalkDesc) % 8 == 0


def test_cabi_argument_errors_do_not_abort():
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    n = C.c_int64(0)
    assert lib.gg_walk_scratch_bytes(0, C.byref(n)) != 0       # bad max_cand -> error code + message
    assert b"gg_walk_scratch_bytes" in lib.gg_last_error()
    assert lib.gg_walk_sample(None, None) != 0
    assert lib.gg_pair_grad(7, 1, 0, None, None, None, None, None, 32, C.c_float(0), None, None, None, None, None, None) != 0
    with pytest.raises(_cabi.GGError):
        _cabi.check(lib.gg_bfs_build(10, 20, None, None, 1, None, None, 2, None, 0, None), "gg_bfs_build")
    with pytest.raises(_cabi.GGError):
        _cabi.check(lib.gg_bfs_build_ex(10, 20, None, None, None, 1, None, None, 2, None, 0, C.c_float(-1.0), 0, None), "gg_bfs_build_ex")
    assert lib.gg_reverse_entries(10, 20, None, None, None, None, None) != 0
    # scratch of the level-synchronous steps: a pure host-side size computation (no GPU): list records + id slabs
    assert lib.gg_walk_flat_bytes(1000, 128, 4, C.byref(n)) == 0 and n.value >= 1000 * (3 * 16 + 2 * 4 + 128 * 4)
    assert lib.gg_walk_flat_bytes(1000, 0, 4, C.byref(n)) != 0 and lib.gg_walk_flat_bytes(1000, 128, 99, C.byref(n)) != 0


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "graphgan_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, flags=re.M), f
                assert "libgg_oracle" not in src and not re.search(r"#include\s*[<\"][^>\"]*oracle", src), f


@pytest.mark.parametrize("name", ["tiny", "rand300", "rand1200", "cagrqc"])
def test_host_graph_equals_reference_reader(name):
    """graph containers vs the dict the reference's utils.read_edges built (stored in the fixture)."""
    from graphgan_b200 import graph as G
    from oracle import canonical as can
    c = loader.load(name)
    hg = G.HostGraph(c.train_edges, c.test_edges)
    assert hg.n_node == c.n
    ptr, flat = can.raw_csr(c.graph)
    assert np.array_equal(hg.raw_indptr, ptr) and np.array_equal(hg.raw_adj, flat)
    for i in (0, c.n // 2, c.n - 1):
        assert hg.neighbors(i).tolist() == c.graph[i]
    ip, adj = can.unique_csr(c.graph)
    assert np.array_equal(hg.indptr, ip) and np.array_equal(hg.adj, adj)
    assert np.array_equal(hg.degrees(), np.diff(ptr))


def test_edge_file_round_trip(tmp_path):
    from graphgan_b200 import graph as G
    c = loader.load("tiny")
    tr, te = tmp_path / "train.txt", tmp_path / "test.txt"
    tr.write_text("".join("%d\t%d\n" % (a, b) for a, b in c.train_edges))
    te.write_text("".join("%d %d\n" % (a, b) for a, b in c.test_edges))
    hg = G.HostGraph.from_files(str(tr), str(te))
    assert hg.n_node == c.n and [hg.neighbors(i).tolist() for i in range(c.n)] == c.graph
    # without the test file node 9 is unknown, so ids are no longer 0..n-1: refuse instead of indexing out of range
    with pytest.raises(ValueError):
        G.HostGraph.from_files(str(tr), "")


def test_config_surface_is_the_references():
    from graphgan_b200 import config
    ref_names = ["modes", "batch_size_gen", "batch_size_dis", "lambda_gen", "lambda_dis", "n_sample_gen", "lr_gen",
                 "lr_dis", "n_epochs", "n_epochs_gen", "n_epochs_dis", "gen_interval", "dis_interval", "update_ratio",
                 "load_model", "save_steps", "n_emb", "multi_processing", "window_size", "app", "dataset",
                 "train_filename", "test_filename", "test_neg_filename", "pretrain_emb_filename_d",
                 "pretrain_emb_filename_g", "emb_filenames", "result_filename", "cache_filename", "model_log"]
    for n in ref_names:
        assert hasattr(config, n), n
    # defaults of src/GraphGAN/config.py:1-41
    assert (config.batch_size_gen, config.batch_size_dis, config.n_sample_gen, config.n_emb, config.window_size) == (64, 64, 20, 50, 2)
    assert (config.lambda_gen, config.lambda_dis, config.lr_gen, config.lr_dis) == (1e-5, 1e-5, 1e-3, 1e-3)
    assert (config.n_epochs, config.n_epochs_gen, config.n_epochs_dis, config.gen_interval, config.dis_interval) == (20, 30, 30, 30, 30)
    assert config.update_ratio == 1 and config.load_model is False and config.save_steps == 10
    assert config.train_filename == "../../data/link_prediction/CA-GrQc_train.txt"
    assert config.emb_filenames == ["../../results/link_prediction/CA-GrQc_gen_.emb", "../../results/link_prediction/CA-GrQc_dis_.emb"]
    assert config.modes == ["gen", "dis"]


def test_flat_dropin_modules_resolve():
    """``import config / generator / discriminator`` from src/GraphGAN (graph_gan.py:8-10)."""
    import importlib
    import sys
    d = os.path.join(ROOT, "src", "GraphGAN")
    sys.path.insert(0, d)
    try:
        for m in ("config", "generator", "discriminator"):
            sys.modules.pop(m, None)
        cfg = importlib.import_module("config")
        gen = importlib.import_module("generator")
        dis = importlib.import_module("discriminator")
        from graphgan_b200 import config as pkg_cfg
        assert cfg is pkg_cfg and gen.Generator.__name__ == "Generator" and dis.Discriminator.__name__ == "Discriminator"
        import inspect
        assert list(inspect.signature(gen.Generator.__init__).parameters)[:3] == ["self", "n_node", "node_emd_init"]
        assert list(inspect.signature(dis.Discriminator.__init__).parameters)[:3] == ["self", "n_node", "node_emd_init"]
    finally:
        sys.path.remove(d)
        for m in ("config", "generator", "discriminator"):
            sys.modules.pop(m, None)


def test_embedding_io_and_link_prediction(tmp_path):
    """read/write in the reference formats; the shipped pretrain embeddings score 0.7598 (SURVEY section 4)."""
    from graphgan_b200 import evaluation, io
    c = loader.load("cagrqc")
    p = tmp_path / "e.emb"
    io.write_embeddings(str(p), c.emb_g.astype(np.float32))
    head = p.read_text().split("\n")[0]
    assert head == "5242\t50"
    back = io.read_embeddings(str(p), 5242, 50)
    assert np.array_equal(back.astype(np.float32), c.emb_g.astype(np.float32))
    t, tn = tmp_path / "t.txt", tmp_path / "tn.txt"
    t.write_text("".join("%d\t%d\n" % (a, b) for a, b in c.test_edges))
    tn.write_text("".join("%d\t%d\n" % (a, b) for a, b in c.test_neg_edges))
    acc = evaluation.LinkPredictEval(str(p), str(t), str(tn), 5242, 50).eval_link_prediction()
    assert abs(acc - 0.7598343685300207) < 2e-3


def test_synthetic_generators_are_deterministic_and_clean():
    from graphgan_b200 import graph as G, synth
    for fn in (synth.erdos_renyi, synth.power_law):
        a, b = fn(5000, 10, seed=3), fn(5000, 10, seed=3)
        assert np.array_equal(a, b) and a.shape[1] == 2
        assert (a[:, 0] != a[:, 1]).all()
        lo, hi = np.minimum(a[:, 0], a[:, 1]), np.maximum(a[:, 0], a[:, 1])
        assert len(set(zip(lo.tolist(), hi.tolist()))) == a.shape[0]
        hg = G.HostGraph(a, None, n_node=5000)
        assert np.array_equal(hg.raw_adj, hg.adj)       # no duplicates / self-loops: one CSR serves both roles
    r = synth.pick_roots(hg.degrees(), 100, seed=1)
    assert (np.diff(r) > 0).all() and (hg.degrees()[r] > 0).all()


def test_bench_reference_arm_machinery():
    """bench.py's CPU legs (oracle port on a fork pool): bounded sample, parent arrays built by the pool, one root
    per task, steady-state rate.  Small graph, 2 workers; checks that a pass runs, covers its sample and that the
    pool and the single-process leg agree on the amount of work (same roots -> same number of sampled edges)."""
    import bench
    from graphgan_b200 import graph as G, synth
    n = 3000
    hg = G.HostGraph(synth.power_law(n, 8, seed=2), None, n_node=n)
    emb = synth.embeddings(n, 32, seed=3)
    roots = synth.pick_roots(hg.degrees(), 200, seed=1)
    out = {}
    for workers in (1, 2):
        ref = bench.CpuReference(hg, emb, roots, 0.5, workers)
        try:
            res, dt = ref.run(7)
            out[workers] = (res, len(ref.sample), int(hg.degrees()[ref.sample].sum()))
        finally:
            ref.close()
        assert res["unit"] == "neg_edges/s" and res["value"] > 0 and res["kind"] == "port" and 1 <= res["cores"] <= workers
        assert not os.path.exists(ref.path)
    # every accepted root contributes len(graph[root]) edges; the two legs may sample different root subsets
    for workers, (res, n_sample, deg_sum) in out.items():
        edges = int(re.search(r"\((\d+) neg edges", res["sample"]).group(1))
        assert 0 < edges <= deg_sum and n_sample >= 2


def test_bench_reference_arm_prints_one_json_line():
    """`bench.py --impl reference` (the arm the driver runs beside ours): exactly one line on stdout, valid JSON with
    the contract's keys; runs on the host cores only (no GPU, nothing read from the reference checkout)."""
    import json
    import subprocess
    import sys
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "powerlaw_100k",
                          "--steps", "1", "--warmup", "0", "--roots", "256"], capture_output=True, text=True, timeout=600,
                         cwd=ROOT, env={**os.environ, "CUDA_VISIBLE_DEVICES": ""})
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [ln for ln in out.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1, out.stdout[:500]
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "neg_edges/s" and d["value"] > 0 and d["higher_is_better"] is True
    assert d["steps"] == 1 and d["warmup"] == 0 and d["n_gpus"] == 1
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "neg_edges/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in d["config"] and "R=256" in d["config"]["workload"]
