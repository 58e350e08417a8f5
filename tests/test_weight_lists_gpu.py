"""Every engine checks the length of its weight list against the reads its config makes.

Each handle is built through its Python module with the create symbol wrapped for one call.  The wrapper takes the exact
list the module passes and builds the engine three times: with the list as given (succeeds), with its last tensor
dropped and with one tensor appended (both fail with the engine named).  A failed build gives back every device buffer
it made before it failed.
"""
import ctypes
import re

import pytest
import torch

from tts_b200 import _lib
from test_device_buffers_gpu import (duration_predictor, engine, flow_forward, flow_reverse, forward_tts,
                                     fullband_melgan, glow_tts, hifigan, live_buffers, melgan, multiband_melgan,
                                     overflow, posterior, pwgan, sdp, speaker_encoder, tacotron2, text_encoder, univnet,
                                     vocoder, wavegrad)

pytestmark = pytest.mark.gpu


def hifigan_bf16():
    from tts_b200.hifigan import HifiganGenerator
    net = HifiganGenerator(in_channels=20, out_channels=1, resblock_type="1", resblock_dilation_sizes=[[1, 3, 5]] * 3,
                           resblock_kernel_sizes=[3, 7, 11], upsample_kernel_sizes=[16, 16, 4, 4],
                           upsample_initial_channel=64, upsample_factors=[8, 8, 2, 2], cond_channels=8).eval()
    net.precision = "bf16"
    return vocoder(net)


def tacotron_dca_bn():
    from tts_b200 import tacotron as TC
    return engine(TC.Tacotron(TC.TacotronConfig(num_chars=30, attention_type="dynamic_convolution",
                                                prenet_type="bn")).eval())


def neuralhmm():   # Overflow's engine without the Glow decoder
    from tts_b200 import overflow as OV
    return engine(OV.NeuralhmmTTS(OV.NeuralhmmTTSConfig(num_chars=30)).eval())


HANDLES = [hifigan, hifigan_bf16, flow_reverse, flow_forward, text_encoder, sdp, posterior, duration_predictor,
           speaker_encoder, glow_tts, forward_tts, melgan, multiband_melgan, fullband_melgan, wavegrad, pwgan, univnet,
           overflow, neuralhmm, tacotron2, tacotron_dca_bn]


# every create symbol a module above builds its handle through
CREATE_SYMBOLS = ["b200tts_hifigan_create_ex", "b200tts_flow_create", "b200tts_flow_create_forward",
                  "b200tts_text_encoder_create", "b200tts_sdp_create", "b200tts_posterior_create",
                  "b200tts_duration_predictor_create", "b200tts_speaker_encoder_create", "b200tts_glow_tts_create",
                  "b200tts_forward_tts_create", "b200tts_melgan_create", "b200tts_wavegrad_create",
                  "b200tts_pwgan_create", "b200tts_univnet_create", "b200tts_overflow_create",
                  "b200tts_tacotron2_create", "b200tts_tacotron_create"]


def check_lists(name, real):
    """A stand-in for the create symbol `name`: runs the checks on the list it is given, then the real call."""
    lib = _lib.lib()
    engine_name = re.match(r"b200tts_(\w+?)_create", name).group(1)
    destroy = getattr(lib, f"b200tts_{engine_name}_destroy")
    seen = []

    def build(args, ptrs):
        arr = (ctypes.c_void_p * len(ptrs))(*ptrs)
        out = ctypes.c_void_p()
        # (cfg, weights, num_weights[, precision], out)
        rc = real(args[0], arr, len(ptrs), *args[3:-1], ctypes.byref(out))
        return rc, out

    def wrapper(*args):
        ptrs = list(args[1])[: args[2]]
        n = len(ptrs)
        before = live_buffers()
        rc, out = build(args, ptrs)
        _lib.check(rc, name)
        destroy(out)
        assert live_buffers() == before
        for wrong in (ptrs[:-1], ptrs + [ptrs[0]]):
            rc, out = build(args, wrong)
            assert rc != 0 and not out.value, f"{name} took a list of {len(wrong)} tensors where it reads {n}"
            msg = lib.b200tts_last_error().decode()
            if len(wrong) > n:
                assert re.search(rf"{engine_name}\w*: expected {n} weight tensors, got {n + 1}$", msg), msg
            with pytest.raises(RuntimeError, match=engine_name):
                _lib.check(rc, name)
            assert live_buffers() == before, f"{live_buffers() - before:+d} device buffers after a failed {name}"
        seen.append(n)
        return real(*args)

    return wrapper, seen


@pytest.mark.parametrize("make", HANDLES, ids=[f.__name__ for f in HANDLES])
def test_weight_list_length_is_checked(make, monkeypatch):
    torch.manual_seed(0)
    build, drop = make()
    lib = _lib.lib()
    checked = []
    for name in CREATE_SYMBOLS:
        wrapper, seen = check_lists(name, getattr(lib, name))
        monkeypatch.setattr(lib, name, wrapper)
        checked.append(seen)
    before = live_buffers()
    build()
    torch.cuda.synchronize()
    drop()
    assert live_buffers() == before
    assert sum(len(s) for s in checked) == 1, "the module did not build its handle through exactly one create call"

