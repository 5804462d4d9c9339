"""CPU: the C-ABI library loads and exports every symbol include/dib_b200.h declares; host-side logic
(beta schedule callback, shard arithmetic, Keras-compat objects, display-row selection)."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "dib_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(dib_[a-z_0-9]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from dib_b200 import _lib
    lib = ctypes.CDLL(_lib.library_path() if os.path.exists(_lib.library_path()) else _lib._build.build_library())
    syms = declared_symbols()
    assert len(syms) >= 14
    for s in syms:
        assert hasattr(lib, s), s
    assert set(syms) == set(_lib.SIGNATURES), set(syms) ^ set(_lib.SIGNATURES)
    lib.dib_build_info.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.dib_build_info()


def test_config_struct_matches_header_field_order():
    from dib_b200 import _lib
    text = open(os.path.join(ROOT, "include", "dib_b200.h")).read()
    body = text[text.index("typedef struct dib_config {"):text.index("} dib_config;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"\b([a-z_0-9]+)\s*;", body)
    assert fields == [f[0] for f in _lib.DibConfig._fields_]


def test_compute_without_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import dib_b200
    with pytest.raises(dib_b200.DibError):
        dib_b200.DistributedIBNet([1, 1], [8], [8], 1)
    with pytest.raises(dib_b200.DibError):
        dib_b200.utils.bhattacharyya_dist_mat(np.zeros((2, 2)), np.zeros((2, 2)))


def test_beta_callback_matches_reference_goldens(golden_dir):
    import dib_b200
    z = np.load(os.path.join(golden_dir, "ref_beta_schedule.npz"))
    for tag in ["train_py_defaults", "nb_radial", "bench"]:
        b0, b1, npre, nann = z[tag + "_args"]
        cb = dib_b200.InfoBottleneckAnnealingCallback(b0, b1, int(npre), int(nann))
        got = np.array([cb.beta_at(int(e)) for e in z[tag + "_epochs"]], dtype=np.float32)
        np.testing.assert_array_equal(got, z[tag + "_beta"])


def test_shard_range_partitions_exactly():
    from dib_b200 import parallel
    for n in [0, 1, 7, 8, 65536, 65537]:
        for world in [1, 2, 3, 8]:
            spans = [parallel.shard_range(n, r, world) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            for (a, b), (c, d) in zip(spans, spans[1:]):
                assert b == c
            sizes = [b - a for a, b in spans]
            assert max(sizes) - min(sizes) <= 1


def test_keras_compat_objects():
    import dib_b200
    from dib_b200.keras_compat import resolve_loss
    opt = dib_b200.optimizers.get("adam")
    opt.learning_rate = 3e-4                                     # train.py:128-129
    assert (opt.beta_1, opt.beta_2, opt.epsilon) == (0.9, 0.999, 1e-7)
    assert resolve_loss(dib_b200.losses.BinaryCrossentropy(from_logits=True)) == "bce_logits"
    assert resolve_loss(dib_b200.losses.SparseCategoricalCrossentropy(from_logits=True)) == "sparse_ce_logits"
    assert resolve_loss("mse") == "mse"
    assert resolve_loss(dib_b200.losses.BinaryCrossentropy()) == "bce_probs"        # Keras default from_logits=False
    with pytest.raises(NotImplementedError):
        resolve_loss(dib_b200.losses.SparseCategoricalCrossentropy())
    sgd = dib_b200.optimizers.get("sgd")
    assert (sgd.learning_rate, sgd.momentum, sgd.nesterov) == (0.01, 0.0, False) and sgd.hyper() == (0.0, 0.0, 0.0)
    rms = dib_b200.optimizers.get("RMSprop")
    assert rms.hyper() == (0.9, 0.0, 1e-7) and dib_b200.optimizers.get(rms) is rms
    with pytest.raises(ValueError):
        dib_b200.optimizers.get("adagrad")
    h = dib_b200.History()
    h.on_epoch_end(0, {"loss": 1.0}); h.on_epoch_end(1, {"loss": 0.5})
    assert h.history == {"loss": [1.0, 0.5]}


def test_select_display_rows():
    from dib_b200 import utils
    raw = np.array([[1.0], [-1.0], [1.0], [-1.0]])
    inds, vals = utils.select_display_rows(raw)
    assert list(vals) == [-1.0, 1.0] and list(raw[inds, 0]) == [-1.0, 1.0]
    raw = np.random.default_rng(0).standard_normal((500, 1))
    inds, vals = utils.select_display_rows(raw, 128, np.random.default_rng(1))
    assert len(inds) == 128 and np.all(np.diff(vals) >= 0) and np.allclose(raw[inds, 0], vals)


def test_bench_accounting_matches_survey_numbers():
    """bench.py's algorithmic work model against SURVEY.md section 8d: C0 forward 600 320 MAC/sample, train
    1 790 720 MAC/sample = 234.7 GFLOP per 65 536-row step; and the ncu traffic lookup parses the committed capture."""
    import importlib.util
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("_bench", os.path.join(root, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    macs, fwd, train = bench.algorithmic_macs(65536)
    assert fwd == 600320 * 65536 and train == 1790720 * 65536
    assert abs(2 * train / 1e9 - 234.7) < 0.05
    assert macs["enc_fused_fwd"] == 16 * 25216 * 65536
    assert macs["enc_fused_bwd"] == 16 * (25216 + 128 * 128 + 128 * 64) * 65536
    t, src = bench.ncu_dram_traffic("enc_fused_bwd")
    assert t is None or (1e6 < t < 1e9 and src.startswith("static: profiles/"))
    cfg = bench.workload_config(2, "fp16", 32768)
    assert cfg["global_batch"] == 65536 and cfg["per_gpu_batch"] == 32768 and cfg["parallelism"] == "dp2"


def test_header_is_plain_c_and_links_from_c(tmp_path):
    """The boundary is a C ABI: include/dib_b200.h must compile as C99 (no C++-isms outside the extern "C" guard) and a C
    program must link against the library and reach a host-only entry point (the CTW estimator needs no GPU)."""
    import os
    import shutil
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = os.path.join(root, "include", "dib_b200.h")
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    subprocess.run([gcc, "-std=c99", "-Wall", "-pedantic", "-Werror", "-fsyntax-only", "-x", "c", hdr], check=True)
    from dib_b200 import _lib
    lib_dir = os.path.dirname(_lib.library_path())
    src = tmp_path / "main.c"
    src.write_text('#include <stdio.h>\n#include "dib_b200.h"\n'
                   'int main(void) { const int8_t s[4] = {1, 0, 0, 1}; double h = 0.0;\n'
                   '  if (dib_ctw_estimate_entropy(s, 4, 2, &h)) { puts(dib_ctw_last_error()); return 1; }\n'
                   '  printf("%.17g %s\\n", h, dib_build_info()); return 0; }\n')
    exe = tmp_path / "main"
    subprocess.run([gcc, "-std=c99", str(src), "-I", os.path.join(root, "include"), "-L", lib_dir, "-ldib_b200",
                    "-Wl,-rpath," + lib_dir, "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    assert float(out[0]) == 1.0232774019241333 and "sm_90a" in " ".join(out[1:])


def test_beta_variable_supports_the_reference_idioms():
    """`kl_loss / model.beta` (train.py:214), `self.beta * tensor` (models.py:118), `beta * 2.0`, float(), np.asarray()."""
    import torch
    from dib_b200.models import _Beta
    b = _Beta(torch.device("cpu"))
    b.assign(0.25)
    assert float(b) == 0.25 and b.value() == np.float32(0.25) and float(np.asarray(b)) == 0.25
    assert b * 2.0 == 0.5 and 2.0 * b == 0.5 and 1.0 / b == 4.0 and b / 0.5 == 0.5 and b + 1 == 1.25 and 1 - b == 0.75
    t = torch.tensor([1.0, 2.0])
    assert torch.equal(b * t, torch.tensor([0.25, 0.5])) and torch.equal(t / b, torch.tensor([4.0, 8.0]))


def test_build_stamp_is_path_independent_and_locked(tmp_path):
    """ADVICE r1: the source stamp must not depend on where the tree lives (the GPU box snapshot is elsewhere)."""
    import importlib.util
    import shutil
    src = os.path.join(ROOT, "distributed-information-bottleneck.github.io_b200")
    dst = tmp_path / "elsewhere" / "pkg"
    os.makedirs(dst.parent / "include")
    shutil.copytree(os.path.join(src, "csrc"), dst / "csrc", ignore=shutil.ignore_patterns("_obj"))
    shutil.copy(os.path.join(src, "build.py"), dst / "build.py")
    shutil.copy(os.path.join(ROOT, "include", "dib_b200.h"), dst.parent / "include" / "dib_b200.h")
    def load(path):
        spec = importlib.util.spec_from_file_location("_b" + str(abs(hash(path))), path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod
    assert load(os.path.join(src, "build.py"))._hash() == load(str(dst / "build.py"))._hash()
