"""CPU: keeps tests/test_gpu_grid_cap.py's KERNELS manifest honest. Every persistent tile kernel of kolibrie_b200/csrc (a __global__
kernel that waits on an mbarrier or takes a tile ticket) must have a capped-grid case there, so that a new tiled kernel cannot arrive
without one; and no launcher may cache a grid size derived from n_sms in a function static, which would fix the first context's grid
for every later one (and make KOLIBRIE_SMS silently miss that kernel)."""
import ast
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kolibrie_b200", "csrc")
GPU_TESTS = os.path.join(ROOT, "tests", "test_gpu_grid_cap.py")

KERNEL_HEAD = re.compile(r"__global__\s+void\s+(?:__launch_bounds__\s*\((?:[^()]|\([^()]*\))*\)\s*)?(\w+)\s*\(")
TICKET = re.compile(r"atomicAdd\s*\(\s*&?\s*[\w.>-]*\b(?:ticket\b|tickets\s*\[|cb\s*\[\s*0\s*\])")
STATIC_INT = re.compile(r"\bstatic\s+(?:const\s+)?(?:int|unsigned|u32|u64|size_t|long(?:\s+long)?)\s+(\w+)\s*=\s*([^;]*);")


def sources():
    out = {}
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh"))):
        with open(path) as f:
            out[os.path.basename(path)] = f.read()
    return out


def body_at(src, start):
    """the brace-balanced body that starts at the first '{' at or after start"""
    i = src.index("{", start)
    depth = 0
    for j in range(i, len(src)):
        depth += {"{": 1, "}": -1}.get(src[j], 0)
        if depth == 0:
            return src[i:j + 1]
    raise AssertionError("unbalanced braces")


def tiled_kernels():
    """kernel name -> file, for every __global__ kernel whose body waits on an mbarrier or takes a tile ticket"""
    out = {}
    for name, src in sources().items():
        for m in KERNEL_HEAD.finditer(src):
            body = body_at(src, m.end())
            if "mbar_wait(" in body or TICKET.search(body):
                out[m.group(1)] = name
    return out


def manifest():
    """KERNELS and the test functions of test_gpu_grid_cap.py, read without importing it (it needs the GPU package)"""
    with open(GPU_TESTS) as f:
        tree = ast.parse(f.read())
    kernels, tests = None, set()
    for node in tree.body:
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "KERNELS" for t in node.targets):
            kernels = ast.literal_eval(node.value)
        elif isinstance(node, ast.FunctionDef) and node.name.startswith("test_"):
            tests.add(node.name)
    assert kernels is not None, "test_gpu_grid_cap.py defines no KERNELS"
    return kernels, tests


def test_the_parser_finds_the_known_tiled_kernels():
    found = tiled_kernels()
    for k in ("scan_kernel", "scan_star_kernel", "probe_index_kernel", "probe_fast_kernel", "probe_direct_kernel", "probe_chained_kernel",
              "probe_grouped_kernel", "quoted_match_kernel", "shuffle_scatter_kernel", "derive_partition_kernel", "derive_probe_kernel"):
        assert k in found, k
    assert "group_kernel" not in found and "build_direct_kernel" not in found, "grid-stride kernels are not tiled"


def test_every_tiled_kernel_has_a_capped_grid_case():
    kernels, tests = manifest()
    missing = sorted(k for k in tiled_kernels() if not kernels.get(k))
    assert not missing, f"tiled kernels without a case in test_gpu_grid_cap.py KERNELS: {missing}"


def test_the_manifest_names_real_kernels_and_tests():
    kernels, tests = manifest()
    everything = "\n".join(sources().values())
    for k, ids in kernels.items():
        assert re.search(r"__global__[^;{]*\b" + k + r"\s*\(", everything), f"KERNELS names {k}, which is no kernel of csrc"
        for t in ids:
            assert t in tests, f"KERNELS[{k!r}] names {t}, which is no test of test_gpu_grid_cap.py"


def test_no_function_static_caches_a_value_of_n_sms():
    bad = []
    for name, src in sources().items():
        for m in STATIC_INT.finditer(src):
            if "n_sms" in m.group(2):
                bad.append(f"{name}: static {m.group(1)} = {m.group(2)}")
        # a static assigned later in the function it is declared in (static int x = 0; if (!x) x = f(n_sms);)
        for m in STATIC_INT.finditer(src):
            var = m.group(1)
            tail = src[m.end():m.end() + 2000]
            end = tail.find("\n}")
            scope = tail[:end if end >= 0 else len(tail)]
            for a in re.finditer(r"(?<![\w.>])" + var + r"\s*=(?!=)\s*([^;]*);", scope):
                if "n_sms" in a.group(1):
                    bad.append(f"{name}: static {var} = {a.group(1)}")
    assert not bad, f"function statics derived from n_sms fix the first context's grid for every later context: {bad}"
