"""CPU test of the C boundary of the tanh RNN's tensor-core policy step: ic3_policy_packed grew by one pointer
(rnn_img); its ctypes mirror must have the header's size and field offsets."""
import ctypes
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_policy_packed_layout_matches_header(tmp_path):
    from ic3net_b200 import _lib
    fields = [f for f, _ in _lib.PolicyPacked._fields_]
    assert fields[-1] == "rnn_img"
    src = open(os.path.join(ROOT, "include", "ic3net_b200.h")).read()
    body = re.search(r"typedef struct \{((?:(?!typedef struct).)*?)\} ic3_policy_packed;", src, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert re.findall(r"\b(\w+);", body) == fields            # same members, same order
    prog = '#include <stdio.h>\n#include <stddef.h>\n#include "ic3net_b200.h"\nint main(){' + \
           'printf("%zu\\n", sizeof(ic3_policy_packed));' + \
           "".join('printf("%%zu\\n", offsetof(ic3_policy_packed, %s));' % f for f in fields) + \
           'printf("%d\\n", IC3_RNN_IMG_BYTES);return 0;}'
    c = tmp_path / "p.c"
    c.write_text(prog)
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(tmp_path / "p")])
    out = [int(v) for v in subprocess.check_output([str(tmp_path / "p")]).decode().split()]
    assert out[0] == ctypes.sizeof(_lib.PolicyPacked)
    assert out[1:-1] == [getattr(_lib.PolicyPacked, f).offset for f in fields]
    assert out[-1] == _lib.RNN_IMG_BYTES


def test_workspace_and_step_validate_the_tanh_configuration(built_lib):
    """Host-side checks only (nothing is launched): the in-scope tanh configuration reports a workspace; a weight image on
    a configuration outside the scope is refused as unsupported."""
    from ic3net_b200 import _lib
    lib = _lib.load()
    hd = (ctypes.c_int32 * _lib.MAX_HEADS)(5, 0, 0, 0)
    pol = dict(B=4, N=3, H=128, O=29, nheads=1, head_dim=hd, hard_attn=0, comm_avg=1, comm_mask_zero=1, env_id0=0, seed=1,
               obs_off=0, obs_vocab=0, obs_ncount=0, cell=_lib.CELL_TANH, passes=1, x_tanh=0, h_from_x=0)
    assert lib.ic3_policy_workspace_bytes(ctypes.byref(_lib.PolicyCfg(**pol))) > 0
    fake = 0x1000                      # never dereferenced: validation fails first
    w = _lib.PolicyPacked(**{f: fake for f, _ in _lib.PolicyPacked._fields_})
    io = _lib.PolicyIO(x=fake, h=fake, h_out=fake, value=fake, logp=fake, workspace=fake)
    for bad in (dict(comm_mask_zero=0), dict(passes=2), dict(x_tanh=1, h_from_x=1), dict(H=64)):
        cfg = _lib.PolicyCfg(**dict(pol, **bad))
        assert lib.ic3_policy_step(ctypes.byref(cfg), ctypes.byref(w), ctypes.byref(io), None) == -3, bad
