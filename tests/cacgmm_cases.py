"""
Shared checks of the CACGMM mask estimator and the permutation aligner (setk_cacgmm_masks,
setk_cacgmm_stft, setk_permu_align), used by the CPU execution model tier (test_cacgmm.py) and the
GPU tier (test_gpu_cacgmm.py).
"""
import hashlib
import json
import os

import numpy as np
import torch

import parity_cases as pc
from oracle import cacgmm_oracle as ao
from oracle import stft_oracle as so
from setk_b200 import plan as P
from setk_b200.libs.cluster import permu_aligner

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL_CACGMM = pc.TOL_CGMM      # fp64 kernels vs the float64 oracle on the same STFT
MARGIN = 1e-9                 # every alignment decision of a case is clearer than this


def check_cacgmm(device, rng, B, C, N, frame_len=512, K=2, iters=3, start="random", update_alpha=True,
                 n_samples=None, permu=False, hop=256):
    """
    setk_cacgmm_masks vs oracle.cacgmm_oracle fed the library's own STFT.  start "random": given fp64
    posteriors; "cgmm": cgmm_init (K = 2).  With permu, the aligned masks must equal the unaligned ones
    gathered through the oracle's mapping of the oracle posteriors.  Returns the worst |diff|.
    """
    x = pc.structured_audio(rng, B, C, N)
    pl = P.StftPlan(C, frame_len, hop, True, True, "hann", B, N, device)
    xt = torch.from_numpy(x).to(device)
    ns = None if n_samples is None else torch.tensor(n_samples, dtype=torch.int32, device=device)
    X = pl.stft(xt, n_samples=ns).cpu().numpy()                    # (B, C, F, T)
    T, F = X.shape[-1], X.shape[2]
    init = None
    if start == "random":
        g = rng.uniform(size=(B, K, T, F))
        init = g / g.sum(1, keepdims=True)
    kw = dict(init_gamma=None if init is None else torch.from_numpy(init).to(device), cgmm_init=start == "cgmm",
              update_alpha=update_alpha, n_samples=ns)
    masks, status = pl.cacgmm_masks(xt, K, iters, **kw)
    masks = masks.cpu().numpy()
    assert masks.shape == (B, K, T, F) and masks.dtype == np.float32
    assert int(status.cpu().abs().sum()) == 0
    aligned = None
    if permu:
        aligned, st2 = pl.cacgmm_masks(xt, K, iters, permu_plan=P.PERMU_PLANS[F], **kw)
        aligned = aligned.cpu().numpy()
        assert int(st2.cpu().abs().sum()) == 0
    worst = 0.0
    for b in range(B):
        Tb = T if n_samples is None else pl.num_frames(int(n_samples[b]))
        gamma = None if init is None else np.transpose(init[b, :, :Tb], (0, 2, 1))
        post = ao.cacgmm_posteriors(X[b][:, :, :Tb], K, iters, gamma=gamma, cgmm_init=start == "cgmm",
                                    update_alpha=update_alpha)
        ref = np.transpose(post, (0, 2, 1))
        err = float(np.max(np.abs(masks[b, :, :Tb] - ref)))
        assert err <= TOL_CACGMM, f"cacgmm masks differ by {err}"
        assert np.all(masks[b, :, Tb:] == 0)
        worst = max(worst, err)
        if permu:
            _, mapping, margins = ao.permu_align(ref)
            assert margins.size == 0 or margins.min() > MARGIN, f"near-tie {margins.min()}"
            assert np.array_equal(aligned[b, :, :Tb], gather(masks[b, :, :Tb], mapping))
            assert np.all(aligned[b, :, Tb:] == 0)
    pl.close()
    return worst


def gather(masks, mapping):
    """masks K x T x F re-ordered per bin: slot k of bin f takes class mapping[k, f]."""
    F = masks.shape[-1]
    return masks[mapping, :, np.arange(F)[None, :]].transpose(0, 2, 1)


def scrambled_masks(rng, B, K, T, F):
    """Per-class activity over time, common to every bin, with the classes of each bin shuffled (B x K x T x F)."""
    out = np.empty((B, K, T, F))
    for b in range(B):
        act = (rng.uniform(size=(K, T)) > 0.5).astype(np.float64) + 0.05
        m = np.repeat(act[:, :, None], F, axis=2) + 0.02 * rng.uniform(size=(K, T, F))
        m /= m.sum(0, keepdims=True)
        for f in range(F):
            out[b, :, :, f] = m[rng.permutation(K), :, f]
    return out


def check_aligner(device, masks, n_frames=None):
    """
    plan.permu_align of fp64 masks (B, K, T, F) vs the host permu_aligner on each utterance's own frames:
    the same mapping on every bin (the oracle's mapping, whose aligned masks are the host's), the
    aligned masks equal to the float32 masks gathered by it, zeros past n_frames.  Returns the
    smallest decision margin.
    """
    B, K, T, F = masks.shape
    nf = None if n_frames is None else torch.tensor(n_frames, dtype=torch.int32, device=device)
    out, mapping = P.permu_align(torch.from_numpy(masks).to(device), n_frames=nf)
    out, mapping = out.cpu().numpy(), mapping.cpu().numpy()
    smallest = np.inf
    for b in range(B):
        Tb = T if n_frames is None else int(n_frames[b])
        ref, ref_map, margins = ao.permu_align(masks[b, :, :Tb])
        assert np.array_equal(ref, permu_aligner(masks[b, :, :Tb]))
        assert margins.size == 0 or margins.min() > MARGIN, f"near-tie {margins.min()}"
        smallest = min(smallest, margins.min() if margins.size else np.inf)
        assert np.array_equal(mapping[b], ref_map), f"utterance {b}: {np.sum(mapping[b] != ref_map)} slots differ"
        assert np.array_equal(out[b, :, :Tb], gather(masks[b, :, :Tb].astype(np.float32), ref_map))
        assert np.all(out[b, :, Tb:] == 0)
    return smallest


# ------------------------------------------------------------------ the reference's fixture ---
def fixture():
    return np.load(os.path.join(GOLD, "ref_cacgmm.npz"))


def fixture_runs(g):
    return sorted({k.split("/")[0] for k in g.files if not k.startswith("in/")})


def fixture_flags(g, name):
    return json.loads(str(g[f"{name}/flags"])), json.loads(str(g[f"{name}/keys"]))


def _fixture_utterances(g, name):
    """(key, C x N float32 audio, K x T x F float64 start or None, options) of every utterance the
    fixture run `name` trained, the random starts drawn from the seed stream as the reference draws them."""
    from oracle.make_golden_cacgmm import parse_flags
    flags, keys = fixture_flags(g, name)
    o = parse_flags(flags)
    np.random.seed(o["seed"])
    K = o["num_classes"]
    for i, key in enumerate(keys):
        if name == "skip" and i == 0:
            continue
        x = so.float_from_pcm16(g[f"in/{key}"])
        T, F = x.shape[1] // 256 + 1, 257            # n_fft 512, hop 256, centred
        init = None
        if o["init_mask"]:
            init = g["noisy/masks/noisy"].astype(np.float64)
        elif not (o["cgmm_init"] and K == 2):
            u = np.random.uniform(size=[K, F, T])
            init = np.transpose(u / np.sum(u, 0, keepdims=True), (0, 2, 1))
        yield key, x, init, o


def _kw(device, init, o):
    return dict(init_gamma=None if init is None else torch.from_numpy(np.ascontiguousarray(init[None])).to(device),
                cgmm_init=o["cgmm_init"], update_alpha=o["update_alpha"],
                permu_plan=P.PERMU_PLANS[257] if o["solve_permu"] else None)


def fixture_from_audio(device, g, name):
    """{key: K x T x F float32} of the fixture run `name` from its audio through plan.cacgmm_masks."""
    out = {}
    for key, x, init, o in _fixture_utterances(g, name):
        C, N = x.shape
        pl = P.StftPlan(C, 512, 256, True, True, "hann", 1, N, device)
        masks, status = pl.cacgmm_masks(torch.from_numpy(x[None]).to(device), o["num_classes"], o["num_iters"],
                                        **_kw(device, init, o))
        pl.close()
        assert int(status.cpu().abs().sum()) == 0
        out[key] = masks[0].cpu().numpy()
    return out


def check_fixture_reference_stft(device, g, name, mean_tol=1e-5, max_tol=5e-3):
    """
    The fixture run `name` with the kernels fed the reference's own complex64 STFT (setk_cacgmm_stft)
    vs the reference's masks.  A flipped bin (|diff| near 1) fails the max bound.  Returns [(mean, max)].
    """
    res = []
    for key, x, init, o in _fixture_utterances(g, name):
        obs = so.multichannel_stft(x, frame_len=512, frame_hop=256, round_power_of_two=True, center=True,
                                   window="hann", transpose=False, out_dtype=np.complex64)
        masks, status = P.cacgmm_from_stft(torch.from_numpy(obs[None]).to(device), o["num_classes"], o["num_iters"],
                                           **_kw(device, init, o))
        assert int(status.cpu().abs().sum()) == 0
        d = np.abs(masks[0].cpu().numpy() - g[f"{name}/masks/{key}"])
        assert d.mean() <= mean_tol and d.max() <= max_tol, (name, key, float(d.mean()), float(d.max()))
        res.append((float(d.mean()), float(d.max())))
    return res


def check_from_audio(device, g, name, tol=TOL_CACGMM):
    """
    The fixture run `name` from its audio (tile STFT + EM + alignment) vs the oracle fed the same
    float32 STFT, then the distance to the reference's masks, which is returned, not bounded: the
    unit-norm observations give a near-silent bin the weight of any other, so the tile STFT's float32
    rounding, which is relative to the frame's energy, moves such bins' directions, and 20 EM
    iterations on 32 frames amplify that (DESIGN.md K16).  Returns [(mean, max)] per utterance.
    """
    res = []
    got = fixture_from_audio(device, g, name)
    for key, x, init, o in _fixture_utterances(g, name):
        C, N = x.shape
        pl = P.StftPlan(C, 512, 256, True, True, "hann", 1, N, device)
        X = pl.stft(torch.from_numpy(x[None]).to(device))[0].cpu().numpy()
        pl.close()
        post = ao.cacgmm_posteriors(X, o["num_classes"], o["num_iters"],
                                    gamma=None if init is None else np.transpose(init, (0, 2, 1)),
                                    cgmm_init=o["cgmm_init"], update_alpha=o["update_alpha"])
        ref = np.transpose(post, (0, 2, 1))
        if o["solve_permu"]:
            ref = ao.permu_align(ref)[0]
        err = float(np.abs(got[key] - ref).max())
        assert err <= tol, (name, key, err)
        d = np.abs(got[key] - g[f"{name}/masks/{key}"])
        res.append((float(d.mean()), float(d.max())))
    return res


def write_fixture_inputs(g, tmp, keys, name="in"):
    """The fixture's utterances as 16-bit wavs under tmp and an scp naming them; returns the scp path."""
    import scipy.io.wavfile as wavfile
    scp = os.path.join(tmp, name + ".scp")
    with open(scp, "w") as f:
        for k in keys:
            path = os.path.join(tmp, k + ".wav")
            wavfile.write(path, 16000, np.ascontiguousarray(g[f"in/{k}"].T))
            f.write(f"{k} {path}\n")
    return scp


def run_cli_case(g, name, tmp, library, device):
    """
    scripts/sptk/estimate_cacgmm_masks.py with the fixture run's flags on its audio: the files hold the
    library's masks from audio with the reference's seed stream (fixture_from_audio), bit for bit, in
    the reference's K x T x F float32 layout; a skipped key's file is left as it was.
    """
    from script_runner import run_script
    flags, keys = fixture_flags(g, name)
    scp = write_fixture_inputs(g, tmp, keys)
    dst = os.path.join(tmp, "out_" + name)
    os.makedirs(dst, exist_ok=True)
    if name == "skip":
        np.save(os.path.join(dst, keys[0] + ".npy"), np.zeros(1, np.float32))
    flags = list(flags)
    if "@noisy" in flags:
        np.save(os.path.join(tmp, "init_noisy.npy"), g["noisy/masks/noisy"])
        with open(os.path.join(tmp, "init.scp"), "w") as f:
            f.write(f"noisy {os.path.join(tmp, 'init_noisy.npy')}\n")
        flags[flags.index("@noisy")] = os.path.join(tmp, "init.scp")
    run_script("estimate_cacgmm_masks.py", [*flags, scp, dst], library=library)
    want = fixture_from_audio(device, g, name)
    for k in keys[1:] if name == "skip" else keys:
        m = np.load(os.path.join(dst, k + ".npy"))
        assert m.dtype == np.float32 and m.shape == g[f"{name}/masks/{k}"].shape
        assert np.array_equal(m, want[k]), (name, k)
    if name == "skip":
        assert np.load(os.path.join(dst, keys[0] + ".npy")).shape == (1,)


# ------------------------------------------------------------------ CGMM outputs unchanged ---
def cgmm_digests(device):
    """
    sha256 of setk_cgmm_masks outputs for the three CGMM cases of test_emu_kernels.test_cgmm_masks
    and of setk_cgmm_stft on the first case's STFT: CGMM shares its kernels with the CACGMM.
    """
    out = {}
    for C, fl, K, init, alpha in ((4, 512, 2, False, False), (3, 1024, 3, True, True), (9, 512, 2, False, False)):
        rng = np.random.default_rng(80 + C)
        B, N, iters = (1, 2800, 2) if C == 9 else (2, 4600, 3)
        ns = torch.tensor([4600, 3300], dtype=torch.int32) if C == 3 else None
        x = pc.structured_audio(rng, B, C, N)
        pl = P.StftPlan(C, fl, 256, True, True, "hann", B, N, device)
        xt = torch.from_numpy(x).to(device)
        X = pl.stft(xt, n_samples=ns)
        T, F = X.shape[-1], X.shape[2]
        ig = None
        if init:
            g = rng.uniform(0.05, 1.0, size=(B, K, T, F))
            ig = torch.from_numpy((g / g.sum(1, keepdims=True)).astype(np.float32)).to(device)
        m, _ = pl.cgmm_masks(xt, K, iters, init_gamma=ig, update_alpha=alpha, n_samples=ns)
        out[f"masks/C{C}"] = hashlib.sha256(m.cpu().numpy().tobytes()).hexdigest()
        if C == 4:
            m, _ = P.cgmm_from_stft(X, K, iters)
            out[f"stft/C{C}"] = hashlib.sha256(m.cpu().numpy().tobytes()).hexdigest()
        pl.close()
    return out
