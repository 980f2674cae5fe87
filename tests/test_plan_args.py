"""
setk_b200.plan's argument checks: a malformed tensor raises before any kernel is launched (the kernels
trust the sizes they are given), an input of another dtype, layout or device is converted to what the
call takes, and a caller's output buffer is used as given or refused.
"""
import numpy as np
import pytest
import torch

from setk_b200 import _lib, plan as P

B, C, F, T, D = 2, 3, 9, 20, 5


def _cplx(*shape, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.complex(torch.randn(shape, generator=g), torch.randn(shape, generator=g))


def _cov(*shape, seed=0):
    """Hermitian positive definite (..., C, C) complex64 matrices."""
    a = _cplx(*shape, seed=seed)
    return a @ a.conj().transpose(-1, -2) + shape[-1] * torch.eye(shape[-1])


def _stft():
    return _cplx(B, C, F, T, seed=1)


def _mask(*shape):
    return torch.rand(shape, generator=torch.Generator().manual_seed(2))


def _rooms(**one):
    """(room, beta, source, receivers) of two problems, one of them given for a single problem only."""
    args = dict(room=np.tile([5.0, 4.0, 3.0], (2, 1)), beta=np.full((2, 6), 0.5),
                source=np.tile([1.0, 1.0, 1.0], (2, 1)), receivers=np.tile([[2.0, 2.0, 1.0]], (2, 1, 1)))
    args.update(one)
    return args["room"], args["beta"], args["source"], args["receivers"]


# every call: a malformed input (or a caller's out= buffer) that no kernel may see
REFUSED = {
    "covariance_mask": (ValueError, lambda: P.covariance(_stft(), _mask(B, T - 8, F))),
    "covariance_mask_ft": (ValueError, lambda: P.covariance(_stft(), _mask(B, T, F), mask_ft=True)),
    "weights_Rs_not_square": (ValueError, lambda: P.weights(_lib.BF_MVDR, _cplx(B, F, C, C - 1), _cov(B, F, C, C))),
    "weights_Rn": (ValueError, lambda: P.weights(_lib.BF_MVDR, _cov(B, F, C, C), _cov(B, F - 4, C, C))),
    "ban_Rn": (ValueError, lambda: P.ban(_cplx(B, F, C), _cov(B, F - 4, C, C))),
    "rank1_Rn": (ValueError, lambda: P.rank1(_cov(B, F, C, C), _cov(B, F - 4, C, C))),
    "apply_weights_weight": (ValueError, lambda: P.apply_weights(_stft(), _cplx(B, F, C - 1))),
    "apply_weights_post_mask": (ValueError, lambda: P.apply_weights(_stft(), _cplx(B, F, C), _mask(B, T - 8, F))),
    "pcm16_to_float_float32": (ValueError, lambda: P.pcm16_to_float(torch.zeros(2, 100))),
    "cm_masks_out_dtype": (ValueError, lambda: P.cm_masks(torch.zeros((B, 64), dtype=torch.uint8), 4, 3,
                                                          out=torch.empty((B, 4, 3), dtype=torch.float64))),
    "cm_masks_out_shape": (ValueError, lambda: P.cm_masks(torch.zeros((B, 64), dtype=torch.uint8), 4, 3,
                                                          out=torch.empty((B, 4, 2)))),
    "gcc_phat_out_dtype": (ValueError, lambda: P.gcc_phat(_cplx(T, F), _cplx(T, F, seed=1), np.zeros(F), np.zeros(D),
                                                          out=torch.zeros((T, D)))),
    "gcc_phat_out_shape": (ValueError, lambda: P.gcc_phat(_cplx(T, F), _cplx(T, F, seed=1), np.zeros(F), np.zeros(D),
                                                          out=torch.zeros((T - 1, D), dtype=torch.float64))),
    "rir_image_unbatched_beta": (ValueError, lambda: P.rir_image(*_rooms(beta=np.full(6, 0.5)), 64, device="cpu")),
    "rir_image_unbatched_source": (ValueError, lambda: P.rir_image(*_rooms(source=[1.0, 1.0, 1.0]), 64, device="cpu")),
    "rir_image_unbatched_receivers": (ValueError, lambda: P.rir_image(*_rooms(receivers=[[2.0, 2.0, 1.0]]), 64,
                                                                      device="cpu")),
    "weights_Rs_real": (TypeError, lambda: P.weights(_lib.BF_MVDR, _cov(B, F, C, C).real, _cov(B, F, C, C).real)),
}


@pytest.mark.parametrize("name", list(REFUSED))
def test_refused_before_launch(emu, name):
    error, call = REFUSED[name]
    launches = _lib.launch_count()
    with pytest.raises(error):
        call()
    assert _lib.launch_count() == launches


def test_converted_inputs_give_the_same_bits(emu):
    stft, mask = _stft(), _mask(B, T, F)
    assert torch.equal(P.covariance(stft, mask.double()), P.covariance(stft, mask))
    assert torch.equal(P.covariance(stft.transpose(2, 3).contiguous().transpose(2, 3), mask),
                       P.covariance(stft, mask))
    w = _cplx(B, C, F, seed=3)
    assert not w.transpose(1, 2).is_contiguous()
    assert torch.equal(P.apply_weights(stft, w.transpose(1, 2), mask.numpy()),
                       P.apply_weights(stft, w.transpose(1, 2).contiguous(), mask))
    wave = torch.linspace(-1.5, 1.5, 301)
    assert torch.equal(P.float_to_pcm16(wave.double()), P.float_to_pcm16(wave))
    room, beta, source, receivers = _rooms()
    assert torch.equal(P.rir_image(room[:1], beta[:1], source[:1], receivers[:1], 64, device="cpu"),
                       P.rir_image(room[0], beta[0], source[0], receivers[0], 64, device="cpu"))
    pcm = P.float_to_pcm16(wave)
    assert torch.equal(P.pcm16_to_float(pcm[::2]), P.pcm16_to_float(pcm[::2].contiguous()))


@pytest.mark.gpu
def test_weights_secondary_input_on_another_gpu(cuda):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    Rs, Rn = _cov(B, 257, 4, 4, seed=4), _cov(B, 257, 4, 4, seed=5)
    w0, st0, _ = P.weights(_lib.BF_MVDR, Rs.to(cuda), Rn.to(cuda))
    w1, st1, _ = P.weights(_lib.BF_MVDR, Rs.to(cuda), Rn.to("cuda:1"))
    assert w1.device == cuda
    assert torch.equal(w0, w1) and torch.equal(st0, st1)
