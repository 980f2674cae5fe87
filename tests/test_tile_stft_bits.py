"""
The chunk-grid tile STFT routes keep their bits: sha256 of every output of the 512- and 1024-point tile
kernels (stft_spill_kernel, stft_spill1024_kernel, feats512_kernel, feats1024_kernel) on the CPU execution
model, against tests/golden/tile_stft_emu_sha256.json.  The grid runs C = 1, 2, 3, 4, 5, 8 (every
channel-group size and both launches of a C > 4 batch), center True and False, a hop that is not a
multiple of 4 (element-wise staging of every tile) and ragged batches whose short utterance fills less
than one tile.  tile_stft_digests(device) runs the same grid on any device.
"""
import hashlib
import json
import os

import numpy as np
import torch

import parity_cases as pc

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# (n_fft, hop, center, C, N, n_samples of a 2-utterance batch or None)
CASES = [
    (512, 256, True, 1, 3000, None),
    (512, 130, True, 2, 3000, None),          # hop % 4 != 0: no tile is bulk-copied
    (512, 256, False, 3, 3000, None),
    (512, 256, True, 4, 3000, [3000, 600]),   # 3 frames: less than one 4-frame tile
    (512, 128, False, 5, 3000, None),
    (512, 256, True, 8, 3000, [3000, 600]),
    (1024, 256, True, 1, 4200, None),
    (1024, 512, False, 2, 4200, None),
    (1024, 256, False, 3, 4200, [4200, 1100]),   # 1 frame: less than one 2-frame tile
    (1024, 128, True, 4, 4200, None),
    (1024, 256, False, 5, 4200, [4200, 1100]),
    (1024, 256, True, 8, 4200, None),
]

# spectral_feats variants: (name, apply_pow, mel, apply_log, sample_scale)
FEATS = [("mag", False, False, False, 1.0), ("pow", True, False, False, 1.0),
         ("mel_log", False, True, True, 1.0), ("pow_mel_scaled", True, True, False, 0.3)]


def _sha(t):
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()


def tile_stft_digests(device):
    """sha256 of StftPlan.stft, spectral_feats and (on the workspace routes) stft_cov for every case."""
    from setk_b200 import plan as P
    from setk_b200.libs.filters import mel
    out = {}
    for n_fft, hop, center, C, N, ns in CASES:
        key = f"{n_fft}/hop{hop}/{'center' if center else 'nocenter'}/C{C}" + ("/ragged" if ns else "")
        rng = np.random.default_rng(n_fft + 10 * hop + C)
        B = 2
        x = torch.from_numpy(pc.structured_audio(rng, B, C, N)).to(device)
        n_samples = torch.tensor(ns, dtype=torch.int32).to(device) if ns else None
        pl = P.StftPlan(C, n_fft, hop, center, True, "hann", B, N, device)
        pl.set_mel(mel(16000, n_fft, n_mels=40 if n_fft == 512 else 80, htk=True))
        out[f"{key}/stft"] = _sha(pl.stft(x, n_samples=n_samples))
        for name, pw, ml, lg, scale in FEATS:
            f = pl.spectral_feats(x, n_samples=n_samples, apply_pow=pw, mel=ml, apply_log=lg, sample_scale=scale)
            out[f"{key}/feats_{name}"] = _sha(f)
        if n_fft == 1024 or C > 4:   # the fused kernel takes C <= 4 at n_fft 512
            T, F = pl.num_frames(N), pl.num_bins
            mask = torch.from_numpy(rng.uniform(size=(B, T, F)).astype(np.float32)).to(device)
            Rs, Rn, maxabs = pl.stft_cov(x, mask, n_samples=n_samples)
            out[f"{key}/Rs"], out[f"{key}/Rn"], out[f"{key}/maxabs"] = _sha(Rs), _sha(Rn), _sha(maxabs)
        pl.close()
    return out


def test_tile_stft_outputs_unchanged(emu):
    want = json.load(open(os.path.join(GOLD, "tile_stft_emu_sha256.json")))["sha256"]
    got = tile_stft_digests(emu)
    assert sorted(got) == sorted(want)
    assert [k for k in want if got[k] != want[k]] == []
