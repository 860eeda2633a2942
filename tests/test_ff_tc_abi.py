"""CPU test of the C boundary of the non-recurrent tanh policies' tensor-core step: ic3_policy_packed grew by one pointer
(ff_img, just in front of rnn_img, the last member); its ctypes mirror must have the header's size and field offsets, and the image size rule
IC3_FF_IMG_BYTES must be that of _lib.ff_img_bytes."""
import ctypes
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [(p, c) for p in range(0, 5) for c in (0, 1)]


def test_policy_packed_layout_and_image_size_match_header(tmp_path):
    from ic3net_b200 import _lib
    fields = [f for f, _ in _lib.PolicyPacked._fields_]
    assert fields[-2:] == ["ff_img", "rnn_img"]
    src = open(os.path.join(ROOT, "include", "ic3net_b200.h")).read()
    body = re.search(r"typedef struct \{((?:(?!typedef struct).)*?)\} ic3_policy_packed;", src, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert re.findall(r"\b(\w+);", body) == fields            # same members, same order
    prog = '#include <stdio.h>\n#include <stddef.h>\n#include "ic3net_b200.h"\nint main(){' + \
           'printf("%zu\\n", sizeof(ic3_policy_packed));' + \
           "".join('printf("%%zu\\n", offsetof(ic3_policy_packed, %s));' % f for f in fields) + \
           "".join('printf("%%zu\\n", IC3_FF_IMG_BYTES(%d, %d));' % pc for pc in CASES) + 'return 0;}'
    c = tmp_path / "p.c"
    c.write_text(prog)
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(tmp_path / "p")])
    out = [int(v) for v in subprocess.check_output([str(tmp_path / "p")]).decode().split()]
    assert out[0] == ctypes.sizeof(_lib.PolicyPacked)
    assert out[1:1 + len(fields)] == [getattr(_lib.PolicyPacked, f).offset for f in fields]
    sizes = out[1 + len(fields):]
    assert sizes == [_lib.ff_img_bytes(p, c) for p, c in CASES]
    # 64 KB (hi + lo of one 128 x 128 fp16 matrix) per weight matrix and pass; passes 0 and 1 are one pass
    assert sizes == [max(1, p) * (2 if c else 1) * 2 * 128 * 128 * 2 for p, c in CASES]


def _policy(**over):
    from ic3net_b200 import _lib
    hd = (ctypes.c_int32 * _lib.MAX_HEADS)(5, 0, 0, 0)
    pol = dict(B=4, N=3, H=128, O=29, nheads=1, head_dim=hd, hard_attn=0, comm_avg=1, comm_mask_zero=0, env_id0=0, seed=1,
               obs_off=0, obs_vocab=0, obs_ncount=0, cell=_lib.CELL_TANH, passes=2, x_tanh=1, h_from_x=1)
    pol.update(over)
    return _lib.PolicyCfg(**pol)


def test_workspace_and_pack_validate_the_configuration(built_lib):
    """Host-side checks only (nothing is launched): one pass reports the nominal 16 bytes, several passes one [B*N, H]
    float32 carry buffer; an ff_img on a configuration outside the non-recurrent tanh step is refused as unsupported."""
    from ic3net_b200 import _lib
    lib = _lib.load()
    assert lib.ic3_policy_workspace_bytes(ctypes.byref(_policy(passes=1))) == 16
    assert lib.ic3_policy_workspace_bytes(ctypes.byref(_policy(passes=3, B=7, N=5))) == 7 * 5 * 128 * 4
    fake = 0x1000                      # never dereferenced: validation fails first
    params = _lib.PolicyParams(encoder_w=fake, encoder_b=fake, c_w=fake, c_b=fake, value_w=fake, value_b=fake,
                               head_w=(ctypes.c_void_p * _lib.MAX_HEADS)(fake, None, None, None),
                               head_b=(ctypes.c_void_p * _lib.MAX_HEADS)(fake, None, None, None),
                               f_w_pass=(ctypes.c_void_p * _lib.MAX_PASSES)(*[fake] * _lib.MAX_PASSES),
                               f_b_pass=(ctypes.c_void_p * _lib.MAX_PASSES)(*[fake] * _lib.MAX_PASSES))
    w = _lib.PolicyPacked(**{f: fake for f, _ in _lib.PolicyPacked._fields_ if f not in ("lstm_img", "bias_cat", "rnn_img")})
    for bad in (dict(x_tanh=0, h_from_x=0), dict(H=64)):
        assert lib.ic3_policy_pack(ctypes.byref(_policy(**bad)), ctypes.byref(params), ctypes.byref(w), None) == -3, bad
