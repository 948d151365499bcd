"""The probe kernels behind benchmarks/hbm_mix.py (ramba_b200/csrc/probe): they stay out of libramba_b200.so, and every
store, walk and load form they time writes exactly `A * s` - a rate measured on a form that writes something else
would be no rate at all."""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..")
CSRC = os.path.join(ROOT, "ramba_b200", "csrc")


def _hbm_mix():
    spec = importlib.util.spec_from_file_location("hbm_mix", os.path.join(ROOT, "benchmarks", "hbm_mix.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_probe_is_not_linked_into_the_library():
    with open(os.path.join(CSRC, "Makefile")) as f:
        mk = f.read()
    objs = re.search(r"^OBJS :=((?:.*\\\n)*.*)$", mk, re.M).group(1)
    assert "build/rb200_api.o" in objs and "probe" not in objs
    assert re.search(r"^probe: ", mk, re.M)
    for name in os.listdir(CSRC):
        if name.endswith((".cu", ".cuh", ".h", ".inc")):
            with open(os.path.join(CSRC, name)) as f:
                assert "probe/" not in f.read(), name


def test_every_arm_is_one_the_probe_accepts():
    # rb200_probe_run: forms 0-2, walks 0-1, 0-3 CTAs/SM (0: one per tile), 1 or 3 outputs, ring depth 2-8; the direct
    # load form only with plain stores and the round-robin walk, at up to 8 CTAs/SM and with an optional resident cap
    for name, arm in _hbm_mix().ARMS.items():
        form, walk, minb, n_out, depth, load, resident = (arm + (0,))[:7]
        assert form in (0, 1, 2) and walk in (0, 1) and n_out in (1, 3) and 2 <= depth <= 8, name
        if load == 0:
            assert minb in (0, 1, 2, 3) and resident == 0, name
        else:
            assert load == 1 and form == 0 and walk == 0 and 0 <= minb <= 8 and resident >= 0, name
        assert ("_1r1w" in name) == (n_out == 1), name


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    out = str(tmp_path_factory.mktemp("probe") / "librb200_probe.so")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-o", out,
                           os.path.join(CSRC, "probe", "rb200_hbm_probe.cu")])
    mod = _hbm_mix()
    return mod, mod.probe_lib(out)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1000, 2048, 5 * 2048 + 37, 1000 * 2048 + 1])
def test_every_form_writes_a_times_s(probe, n):
    import torch

    mod, lib = probe
    a = torch.arange(n, dtype=torch.float64, device="cuda") / 1000.0 + 0.25
    outs = [torch.empty_like(a) for _ in range(3)]
    st = torch.cuda.current_stream().cuda_stream
    for name, arm in mod.ARMS.items():
        form, walk, minb, n_out, depth, load, resident = (arm + (0,))[:7]
        for o in outs:
            o.fill_(-1.0)
        rc = lib.rb200_probe_run(form, walk, minb, load, resident, n_out, depth, a.data_ptr(), outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), n, st)
        if rc < 0 and rc > -100:
            continue  # does not fit the asked CTAs per SM (the staged form at 3)
        assert rc == 0, (name, rc)
        torch.cuda.synchronize()
        for j, s in enumerate((1.5, 2.5, 3.5)):
            want = a * s if j < n_out else torch.full_like(a, -1.0)
            assert torch.equal(outs[j], want), (name, j)
