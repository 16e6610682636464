"""INTEGRATION.md shows the one-line `jt.code` bodies a JNeRF maintainer would add for every operator.  Jittor is not available
here, so the stubs cannot run -- but they must at least be valid calls of include/ngp_b200.h: every `NGP_OK(ngp_...(...))`
statement of the document is extracted and type-checked by the host compiler against the real header (argument count, pointer
versus scalar in every position), with Jittor's injected names (`inK_p`, `outK_p`, `inK_shapeJ`, `rng`, ...) declared the way
jt.code declares them."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PREAMBLE = r'''
#include <stdint.h>
#include <stdexcept>
#include "ngp_b200.h"
#define NGP_OK(x) do { if ((x) != 0) throw std::runtime_error(ngp_last_error()); } while (0)
struct AnyPtr { template <class T> operator T*() const { return nullptr; } };       // a typed device pointer of any type
struct Rng { uint64_t state, inc; };                                                // jittor::rng (pcg32), OPS/global_vars.py
struct Var { uint64_t num; };
static inline uint32_t NERF_CASCADES() { return 5; }                                // generated header, density_grid_sampler.py:96-106
typedef uint16_t in1_type; typedef uint16_t out_type;
'''


def extract_calls(text):
    calls, i = [], 0
    while True:
        k = text.find("NGP_OK(", i)
        if k < 0:
            return [c for c in calls if "ngp_" in c]
        j, depth = k + 7, 1
        while depth:
            depth += text[j] == "("
            depth -= text[j] == ")"
            j += 1
        calls.append(text[k:j])
        i = j


def _type_check(calls, declared, tmp_path, name):
    body = []
    for n, c in enumerate(calls):
        c = re.sub(r"\{[^{}]*\}", "1", c)                       # python f-string fields become literals
        ids = set(re.findall(r"[A-Za-z_][A-Za-z_0-9]*", re.sub(r"/\*.*?\*/", "", c)))
        ids -= {"NGP_OK", "NGP_F16", "NGP_F32", "NERF_CASCADES", "nullptr", "sizeof", "const", "uint32_t", "uint8_t", "in1_type", "out_type",
                "state", "inc", "num", "f", "e", "float"} | declared
        decl = []
        for v in sorted(ids):
            if v == "rng":
                decl.append("Rng rng{};")
            elif v == "out":
                decl.append("Var out_{}; Var* out = &out_;")
            elif v in ("handle64", "handle64_of_rank_r"):
                decl.append(f"uint8_t {v}[64] = {{0}};")
            elif v in ("offset", "offset_r"):
                decl.append(f"uint64_t {v} = 0;")
            elif v == "peer_base":
                decl.append("void* peer_base[16] = {nullptr};")
            elif v.endswith("_p") or v in ("peer_table", "peer_table_grad", "peer_w_grad", "peer_flags", "m_slice", "v_slice", "master_slice",
                                           "w_param", "w_m", "w_v", "w_master", "my_flags"):
                decl.append(f"AnyPtr {v};")
            elif v in ("lr", "thresh", "aabb0", "aabb1"):
                decl.append(f"float {v} = 0.5f;")
            else:
                decl.append(f"uint32_t {v} = 1;")
        body.append(f"void stub_{n}() {{ {' '.join(decl)} {c}; }}")
    src = tmp_path / name
    src.write_text(PREAMBLE + "\n".join(body) + "\n")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]


def test_every_stub_in_integration_md_type_checks_against_the_header(tmp_path):
    text = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    calls = extract_calls(text)
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ngp_b200.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(ngp_[a-z0-9_]+)\s*\(", hdr))
    used = {re.search(r"(ngp_[a-z0-9_]+)\(", c).group(1) for c in calls}
    assert len(calls) >= 20 and used <= declared
    # every compute entry point of the header has a stub in the document (host helpers and debug aids excepted)
    helpers = {"ngp_last_error", "ngp_version", "ngp_sm_count", "ngp_debug_timeout_flag", "ngp_hash_offsets", "ngp_hash_level_table", "ngp_hash_level_table_primes",
               "ngp_mlp_param_count", "ngp_march_workspace_bytes", "ngp_pcg32_seed", "ngp_pcg32_advance", "ngp_ipc_close", "ngp_raygen",
               "ngp_prepare_batch", "ngp_composite_loss_bwd", "ngp_mlp_bwd_dgrad", "ngp_blend_target"}
    for name in sorted(declared - helpers - used):
        assert name in text, f"{name} is declared in the header but INTEGRATION.md never mentions it"
    assert not (declared - helpers - used), declared - helpers - used
    _type_check(calls, declared, tmp_path, "stubs.cpp")


def test_jittor_glue_module_imports_and_its_cuda_bodies_type_check(tmp_path):
    """jnerf_b200/jittor_glue.py is the importable form of the document: it must import without Jittor, and every cuda_src body it hands
    to jt.code must be a valid call of the header (same check as above, on the module's SRC table)."""
    import sys
    sys.path.insert(0, ROOT)
    from jnerf_b200 import jittor_glue as glue
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ngp_b200.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(ngp_[a-z0-9_]+)\s*\(", hdr))
    calls = extract_calls("\n".join(glue.SRC.values()))
    assert len(calls) == len(glue.SRC) >= 19
    _type_check(calls, declared, tmp_path, "glue.cpp")
    assert "-Xlinker" in next(iter(glue.ngp_options())) and glue.NGP_LIB.endswith("libngp_b200.so")
    import pytest
    try:
        import jittor  # noqa: F401
    except ImportError:
        with pytest.raises(ImportError, match="Jittor"):
            glue.sh_encode(None)
