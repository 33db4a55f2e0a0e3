"""CPU tests of the C-ABI boundary: the library loads, exports every symbol include/rfx.h declares, the ctypes
mirrors have the C layout, and (without a GPU) entry points fail loudly instead of falling back."""
import ctypes as C
import os
import re
import subprocess
import sys

import pytest

from realism_effects_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_the_declared_abi(built):
    """Every rfx_* function include/rfx.h declares is exported and listed in abi.EXPORTS, and the library reports ABI version 3."""
    hdr = open(os.path.join(ROOT, "include", "rfx.h")).read()
    declared = sorted(set(re.findall(r"\b(rfx_[a-z0-9_]+)\s*\(", hdr)))
    assert len(declared) >= 30
    lib = abi.lib()
    missing = [n for n in declared if not hasattr(lib, n)]
    assert not missing, missing
    assert sorted(set(abi.EXPORTS)) == declared
    assert lib.rfx_version() == 3
    assert [lib.rfx_format_bytes(f) for f in range(4)] == [4, 16, 8, 4]


def test_ctypes_struct_layout_matches_c(tmp_path):
    names = {"rfx_plane": abi.Plane, "rfx_camera": abi.CameraS, "rfx_ssgi_params": abi.SsgiParams, "rfx_temporal_params": abi.TemporalParams,
             "rfx_poisson_params": abi.PoissonParams, "rfx_compose_params": abi.ComposeParams, "rfx_hbao_params": abi.HbaoParams,
             "rfx_ao_compose_params": abi.AoComposeParams, "rfx_motion_blur_params": abi.MotionBlurParams, "rfx_env_desc": abi.EnvDesc,
             "rfx_ssgi_chain_options": abi.ChainOptions, "rfx_ssgi_frame": abi.SsgiFrame, "rfx_ssgi_host_frame": abi.SsgiHostFrame}
    src = tmp_path / "sz.c"
    body = "\n".join(f'printf("{n} %zu\\n", sizeof({n}));' for n in names)
    src.write_text(f'#include <stdio.h>\n#include "rfx.h"\nint main(void){{{body} return 0;}}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])  # the header is plain C
    out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    for n, cls in names.items():
        assert int(out[n]) == C.sizeof(cls), (n, out[n], C.sizeof(cls))


def test_no_cpu_fallback_without_gpu(built):
    import torch

    if torch.cuda.is_available():
        pytest.skip("box has a GPU")
    from realism_effects_b200 import engine

    with pytest.raises(abi.RfxError):
        engine.Context(0)  # must fail loudly: there is no CPU path


def test_product_never_imports_oracle():
    """The product package must not reference oracle/ or tests/ (SURVEY tier rule 3)."""
    pkg = os.path.join(ROOT, "realism_effects_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                for bad in ("import orc", "librfx_oracle", "chain_harness", "from tests", "rfx_oracle", "orc_"):
                    assert bad not in txt, (f, bad)


def test_napi_shim_type_checks_against_the_header():
    """js/napi/shim.cc cannot be built here (no Node), but every rfx_* call in it must match include/rfx.h: it is type-checked with
    g++ -fsyntax-only against the real header and a stub of the N-API prototypes (tools/check_shim.sh); and js/index.js exports the
    reference's eight plugin classes (src/index.js:16-31)."""
    import os
    import re
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run(["bash", os.path.join(root, "tools", "check_shim.sh")], capture_output=True, text=True)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr
    js = open(os.path.join(root, "js", "index.js")).read()
    exported = set(re.findall(r"export class (\w+)", js))
    assert {"SSGIEffect", "SSREffect", "TRAAEffect", "MotionBlurEffect", "HBAOEffect", "VelocityDepthNormalPass", "TemporalReprojectPass", "PoissonDenoisePass"} <= exported
    shim = open(os.path.join(root, "js", "napi", "shim.cc")).read()
    bound = set(re.findall(r'FN\("(\w+)"', shim))
    used = set(re.findall(r"rfx\.(\w+)\(", js))
    assert used <= bound, sorted(used - bound)                      # every rfx.<fn> the JS classes call is exported by the shim
    for sig in ("update(renderer, inputBuffer, deltaTime)", "update(renderer, inputBuffer)", "render(renderer)"):
        assert sig in js
