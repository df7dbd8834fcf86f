"""The C-ABI: header <-> ctypes table <-> exported symbols (CPU only, no compute calls)."""
import ctypes
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'fsdet.h')
LIB = os.path.join(ROOT, 'fewshot_detection_b200', 'libfsdet.so')


def parse_header():
    src = open(HEADER).read()
    src = re.sub(r'/\*.*?\*/', ' ', src, flags=re.S)
    decls = {}
    for m in re.finditer(r'(?:^|\n)\s*(int|size_t|const char\*)\s+(fsdet_\w+)\s*\(([^;]*?)\)\s*;', src):
        ret, name, params = m.group(1), m.group(2), m.group(3).strip()
        codes = ''
        if params and params != 'void':
            for prm in params.split(','):
                prm = prm.strip()
                if '*' in prm:
                    codes += 'p'
                elif 'size_t' in prm:
                    codes += 'z'
                elif 'long long' in prm:
                    codes += 'q'
                elif 'double' in prm:
                    codes += 'd'
                elif 'float' in prm:
                    codes += 'f'
                elif 'int' in prm:
                    codes += 'i'
                else:
                    raise AssertionError('unparsed parameter %r in %s' % (prm, name))
        decls[name] = (codes, {'int': 'i', 'size_t': 'z', 'const char*': 's'}[ret])
    return decls


def _build_if_needed():
    if not os.path.exists(LIB):
        import sys
        sys.path.insert(0, ROOT)
        import __graft_entry__
        __graft_entry__.build()


def test_header_matches_ctypes_table():
    _build_if_needed()
    from fewshot_detection_b200 import _lib
    decls = parse_header()
    assert len(decls) >= 30
    assert set(decls) == set(_lib.SIGNATURES), set(decls) ^ set(_lib.SIGNATURES)
    for name, sig in decls.items():
        assert _lib.SIGNATURES[name] == sig, (name, _lib.SIGNATURES[name], sig)


def test_library_exports_every_declared_symbol():
    _build_if_needed()
    lib = ctypes.CDLL(LIB)
    for name in parse_header():
        assert hasattr(lib, name), name
    lib.fsdet_version.restype = ctypes.c_int
    assert lib.fsdet_version() >= 100
    assert lib.fsdet_compiled_arch() == 90
    assert lib.fsdet_num_sms() == 132


def test_library_is_sm90a_native():
    _build_if_needed()
    out = subprocess.run(['cuobjdump', '-lelf', LIB], capture_output=True, text=True).stdout
    assert 'sm_90a' in out, out


def test_product_package_never_imports_the_oracle():
    """oracle/ is test infrastructure: only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import it."""
    pkg = os.path.join(ROOT, 'fewshot_detection_b200')
    offenders = []
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh', '.h')):
                src = open(os.path.join(dirpath, f)).read()
                if re.search(r'^\s*(from|import)\s+oracle\b', src, flags=re.M):
                    offenders.append(os.path.join(dirpath, f))
    assert offenders == []
    for f in os.listdir(os.path.join(ROOT, 'dropin')):
        assert 'oracle' not in open(os.path.join(ROOT, 'dropin', f)).read()


def test_tile_plans_of_the_benchmarked_layers():
    """Host-side planning of the tensor-core kernels at configs[1] (64 query + 20 support images, 416x416) - pure C
    functions of the library, no GPU: which layers the halo-tile kernel takes, how many BatchNorm partial rows the
    kernels emit, and that the weight gradient's split-K fills whole rounds of the 132 SMs."""
    _build_if_needed()
    from fewshot_detection_b200 import _lib
    L = _lib.lib
    halo = {  # (B, H, Cin, Cout) -> taken by the halo kernel (3x3, mode 3)
        (64, 208, 32, 64): 1, (64, 208, 64, 32): 1, (20, 208, 32, 64): 1,      # conv2 forward / input gradient, support twin
        (64, 104, 64, 128): 1, (64, 104, 128, 64): 1, (20, 104, 64, 128): 1,   # conv3 / conv5
        (64, 52, 128, 256): 0,                                                 # width 52 does not tile by 8
        (64, 13, 512, 1024): 0, (64, 26, 256, 512): 0,                         # long K / too many channels
        (2, 104, 64, 128): 0,                                                  # too few tiles for the persistent grid
    }
    for (B, H, Cin, Cout), want in halo.items():
        assert L.fsdet_conv_tc_uses_halo(B, H, H, Cin, Cout, 3, 3) == want, (B, H, Cin, Cout)
        assert L.fsdet_conv_tc_uses_halo(B, H, H, Cin, Cout, 3, 3 | 64) == 0          # mode bit 6: never
        rows = L.fsdet_conv_tc_stat_rows(B, H, H, Cin, Cout, 3, 3)
        assert rows == (132 if want else -(-B * H * H // 128)), (B, H, Cin, Cout, rows)
    assert L.fsdet_conv_tc_uses_halo(64, 208, 208, 32, 64, 1, 3) == 0                 # 1x1
    assert L.fsdet_conv_tc_uses_halo(64, 208, 208, 32, 64, 3, 0) == 0                 # only the 3-term mode
    # weight gradient (fp16 x fp16 mode, 128-wide tiles): CTAs = tiles * splits never spill a few CTAs into an extra round
    for B, H, Cin, Cout in [(64, 208, 64, 64), (64, 104, 64, 128), (64, 52, 128, 256), (64, 26, 256, 512), (64, 13, 512, 1024),
                            (64, 13, 1024, 1024), (64, 13, 1280, 1024), (20, 208, 64, 64), (20, 13, 512, 1024)]:
        taps = 1 if Cin >= 128 else 2
        cib = 128 // taps
        tiles = -(-Cin // cib) * -(-9 // taps) * -(-Cout // 128)
        ws = L.fsdet_conv_tc_wgrad_workspace_floats(B, H, H, Cin, Cout, 3, 0)
        splits = max(1, ws // (Cout * 9 * Cin))
        ctas = tiles * splits
        rounds = -(-ctas // 132)
        assert ctas > 0.8 * rounds * 132 or splits == 1, (B, H, Cin, Cout, tiles, splits, ctas)
