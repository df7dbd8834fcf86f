"""Shared helpers of the host-emulation tests: build a tools/host_emul library with g++ and route
fewshot_detection_b200.image's C-ABI calls to it (CPU tensors, same argument lists)."""
import ctypes
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, 'tools', 'host_emul', 'cuda_host_emul.h')


def build_emul(name, kernel_src, opt='-O2'):
    inc = '/usr/local/cuda/include'
    if not os.path.exists(os.path.join(inc, 'cuda_runtime.h')):
        pytest.skip('CUDA headers not found')
    src = os.path.join(ROOT, 'tools', 'host_emul', name + '_emul.cpp')
    ksrc = os.path.join(ROOT, 'fewshot_detection_b200', 'csrc', kernel_src)
    lib = os.path.join(ROOT, 'build', 'lib%s_emul.so' % name)
    os.makedirs(os.path.dirname(lib), exist_ok=True)
    deps = [src, HDR, ksrc] + [os.path.join(os.path.dirname(HDR), f) for f in os.listdir(os.path.dirname(HDR))]
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(p) for p in deps):
        cmd = ['g++', opt, '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-pthread', '-w',
               '-DFSDET_HOST_EMULATION', '-I' + inc, '-include', HDR, '-x', 'c++', src, '-o', lib]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0, r.stdout
    return ctypes.CDLL(lib)


def route_image_calls_to_emulation(monkeypatch, emul):
    """fewshot_detection_b200.image on CPU tensors: `call(...)` goes to the emulated kernels with the real argument
    lists; default device becomes the CPU."""
    import torch
    from fewshot_detection_b200 import image as I
    V = ctypes.c_void_p

    def fake_call(name, *a):
        if name == 'fsdet_augment_batch':
            src, geom, color, n, W, H, kmax, filt, ws, ws_bytes, out, out_u8, status, stream = a
            L = max(W, H)
            tbytes = n * 2 * L * (2 + kmax) * 4
            assert ws_bytes >= tbytes + n * 768
            emul.emul_augment_batch(V(src), V(geom), V(color), n, W, H, kmax, filt, V(ws), V(ws + tbytes), V(out),
                                    V(out_u8) if out_u8 else None, V(status))
        elif name == 'fsdet_box_masks':
            rects, n, H, W, out, stream = a
            emul.emul_box_masks(V(rects), n, H, W, V(out))
        else:
            raise AssertionError('unexpected C-ABI call %s' % name)
        return 0
    monkeypatch.setattr(I, 'call', fake_call)
    monkeypatch.setattr(I, '_st', lambda: None)
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: True)
    monkeypatch.setattr(I, '_default_device', lambda: torch.device('cpu'))
    return I
