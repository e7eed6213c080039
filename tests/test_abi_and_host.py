"""CPU checks of the product library: it loads, exports every symbol of include/paillier_b200.h, and
refuses loudly to compute without a CUDA device (no CPU fallback)."""
import os
import re

import numpy as np
import pytest

from oracle.golden import H, load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    ge.build()


def test_header_symbols_exported(pkg, built):
    hdr = open(os.path.join(ROOT, "include", "paillier_b200.h")).read()
    declared = set(re.findall(r"\b(pai_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 30
    engine_mod = __import__("importlib").import_module("python-paillier_b200.engine")
    assert declared == set(engine_mod.SYMBOLS), declared ^ set(engine_mod.SYMBOLS)
    eng = pkg.Engine()                      # the CUDA build, loaded through ctypes; binds every symbol
    assert eng.path.endswith("libpaillier_b200.so")
    assert eng.lib.pai_version() >= 100
    assert eng.launch_count() == 0


def test_no_cpu_fallback(pkg, built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is for GPU-less hosts")
    eng = pkg.Engine()
    assert eng.device_count() == 0
    with pytest.raises(pkg.EngineUnavailable):
        pkg.PublicContext(H(load_golden("vectors_256.json")["n"]), engine=eng)
    with pytest.raises(pkg.EngineUnavailable):
        pkg.PrivateContext(293, 433, engine=eng)
    with pytest.raises(pkg.EngineUnavailable):
        pkg.ModContext(2 ** 127 - 1, engine=eng)
    pk = pkg.PaillierPublicKey(H(load_golden("vectors_256.json")["n"]))
    with pytest.raises(pkg.EngineUnavailable):
        pk.encrypt(3)


def test_limb_packing_roundtrip(pkg):
    vals = [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 255 + 12345, 2 ** 512 - 1]
    arr = pkg.ints_to_limbs(vals, 16)
    assert arr.shape == (6, 16) and arr.dtype == np.uint32 and arr[1, 0] == 1 and arr[3, 1] == 1
    assert pkg.limbs_to_ints(arr) == vals
    with pytest.raises(ValueError):
        pkg.ints_to_limbs([2 ** 512], 16)
    with pytest.raises(ValueError):
        pkg.ints_to_limbs([-1], 16)


def test_shard_range(pkg):
    par = __import__("importlib").import_module("python-paillier_b200.parallel")
    for batch in (0, 1, 7, 8, 1000, 4194304):
        for world in (1, 2, 3, 8):
            spans = [par.shard_range(batch, r, world) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == batch
            assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
            sizes = [hi - lo for lo, hi in spans]
            assert max(sizes) - min(sizes) <= 1


def test_build_tracks_every_device_header():
    """A header missing from the staleness lists means an edited kernel silently keeps running from an old .so."""
    import importlib
    import os
    import re
    import __graft_entry__ as ge
    build = importlib.import_module("python-paillier_b200.build")
    csrc = build.CSRC
    included = set()
    for name in os.listdir(csrc):
        with open(os.path.join(csrc, name)) as f:
            included.update(re.findall(r'#include "(pai_[a-z_]+\.(?:cuh|h))"', f.read()))
    assert included and included <= set(build.HEADERS)
    with open(ge.__file__) as f:
        text = f.read()
    assert all('"%s"' % h in text for h in included)


def test_tc_shared_memory_budget(tmp_path):
    """The number of 128-thread groups a tensor-core CTA runs is decided by shared memory (pai_engine.cu: tc_geometry_of
    takes the largest count whose buffers fit 227 KB - 128 B).  Pin the counts the measured numbers rely on, so that a
    buffer growing by a few bytes cannot silently drop a group: 3 groups at 192/256 digits (x1 in the table strip),
    4 groups at 64/128 digits, 1 group at 384 digits."""
    import subprocess
    src = tmp_path / "budget.cpp"
    src.write_text(r'''
#define PAI_HOSTSIM 1
#include <cstdio>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>
#include <algorithm>
#include "%s/python-paillier_b200/csrc/pai_cta.cuh"
using namespace pai;
template <int N> void row() {
  for (int g = 1; g <= 4; g++)
    printf("%%d %%d %%zu %%zu %%zu %%d\n", N, g, tc_enc_smem_bytes<N>(128 * g), tc_pow_smem_bytes<N>(128 * g), tc_dec_smem_bytes<N>(128 * g),
           (int)tc_x1_global<N>());
}
int main() { row<2>(); row<4>(); row<6>(); row<8>(); row<12>(); return 0; }
''' % ROOT)
    exe = tmp_path / "budget"
    subprocess.run(["g++", "-std=c++17", "-x", "c++", str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    limit = 232448 - 128                                   # cudaDevAttrMaxSharedMemoryPerBlockOptin on sm_90 minus the margin
    fits = {}
    for line in out:
        if line.strip():
            n, g, enc, pw, dec, x1g = (int(v) for v in line.split())
            fits[(n, g)] = (enc <= limit, pw <= limit, dec <= limit, x1g)
    best = lambda n, i: max(g for g in range(1, 5) if fits[(n, g)][i])
    assert [fits[(n, 1)][3] for n in (2, 4, 6, 8, 12)] == [0, 0, 1, 1, 0]
    # register budget (BodyMaxThreads) caps 192/256 digits at 3 groups; shared memory has to allow at least that many
    assert best(8, 0) == 3 and best(8, 1) == 3 and best(8, 2) == 2      # 4096-bit-key decrypt: four bands, two groups
    assert best(6, 0) >= 3 and best(6, 1) >= 3 and best(6, 2) >= 3
    assert best(4, 0) == 4 and best(4, 1) == 4 and best(4, 2) == 4
    assert best(2, 0) == 4 and best(2, 2) == 4
    assert best(12, 0) == 1 and best(12, 1) == 1                        # (no 384-digit decrypt: keys stop at 4096 bits)
