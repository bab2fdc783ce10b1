"""WORLD analysis on the GPU (gantts_world_dio / _stonemask / _cheaptrick, gantts_sp2mc, gantts_modspec_smoothing, the
analysis chain and objective --wav-dir) against the numpy restatement oracle.world_analysis_port on seeded ragged batches
of harmonic waveforms (1-5 s, 16 and 48 kHz): frame counts and V/UV identical, f0, sp and mc within the stated fp64
tolerances, every row bit-identical to its B = 1 run under other padding, the status word, a synthesis round trip, and
the command end to end with and without --wav-dir."""
import os

import numpy as np
import pytest
import torch

from oracle import sptk_port
from oracle import world_analysis_port as A

pytestmark = pytest.mark.gpu

FP = 5.0
# Tolerances about 10x the worst seen on an H100 (f0 4e-14, StoneMask 7e-16, log sp 1.3e-8, mc 8e-11):
F0_TOL = 1e-12      # DIO and StoneMask f0, relative: the same arithmetic in the same order but for cos / FFT rounding
SP_TOL = 1e-7       # |log sp - log sp_oracle| on the same f0: CheapTrick differences cumulative sums (see DESIGN)
MC_TOL = 1e-9       # |mc - mc_oracle|, absolute, the mel-cepstra of those envelopes


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__
    __graft_entry__.build()
    return torch.device("cuda:0")


def wave(rng, fs, seconds):
    """int16-valued float64 samples: voiced runs of 80-400 Hz (seven harmonics, f0 drifting) with unvoiced gaps."""
    hop = int(fs * FP / 1000)
    F = int(seconds * 1000 / FP)
    f0 = np.zeros(F)
    j = int(rng.randint(5, 30))
    while j < F:
        run = int(rng.randint(30, 120))
        a, b = rng.uniform(80, 400, 2)
        f0[j:j + run] = np.linspace(a, b, len(f0[j:j + run]))
        j += run + int(rng.randint(10, 50))
    f = np.repeat(f0, hop)
    ph = np.cumsum(2 * np.pi * f / fs)
    x = sum(np.where(f > 0, np.cos(k * ph + k) / k, 0.0) for k in range(1, 8))
    return np.round(np.clip(6000.0 * x + rng.randn(len(f)) * 20.0, -32768, 32767)), f0


def run_chain(dev, waves, fs, order=24, pad=0.0, S=None):
    from gantts_b200 import analysis, generate, ops
    S = S or max(len(w) for w in waves)
    xb = np.full((len(waves), S), pad)
    for i, w in enumerate(waves):
        xb[i, :len(w)] = w
    x = torch.from_numpy(xb).to(dev)
    L = torch.tensor([len(w) for w in waves], dtype=torch.int64, device=dev)
    f0, info = ops.world_dio(x, L, fs, FP)
    rf0 = ops.world_stonemask(x, L, f0, info, fs, FP)
    sp = ops.world_cheaptrick(x, L, rf0, info, fs, FP, generate.cheaptrick_fft_size(fs))
    mc = ops.sp2mc(sp, info[:-1], order, generate.mcep_alpha(fs))
    frames = ops.world_analysis_check(info)
    return frames, f0.cpu().numpy(), rf0.cpu().numpy(), sp.cpu().numpy(), mc.cpu().numpy()


@pytest.mark.parametrize("fs,rows,longest", [(16000, 20, 5.0), (48000, 6, 2.5)])
def test_kernels_against_the_restatement(dev, fs, rows, longest):
    rng = np.random.RandomState(fs + rows)
    waves = [wave(rng, fs, rng.uniform(1.0, longest))[0] for _ in range(rows)]
    frames, f0, rf0, sp, mc = run_chain(dev, waves, fs)
    n = sptk_port.cheaptrick_fft_size(fs)
    alpha = sptk_port.mcepalpha(fs)
    stream = A.randn_stream(frames.max() * (2 * n + 2))
    worst = {"f0": 0.0, "stonemask": 0.0, "logsp": 0.0, "mc": 0.0}
    ties = checked = 0
    for b, x in enumerate(waves):
        F = A.dio_frames(len(x), fs, FP)
        assert frames[b] == F
        assert np.all(f0[b, F:] == 0) and np.all(sp[b, F:] == 0) and np.all(mc[b, F:] == 0)
        want, t, det = A.dio(x, fs, FP, details=True)
        assert np.array_equal(f0[b, :F] > 0, want > 0), b                       # V/UV identical
        v = want > 0
        worst["f0"] = max(worst["f0"], float(np.max(np.abs(f0[b, :F][v] / want[v] - 1), initial=0)))
        # the candidate choice's tie band: voiced frames whose two lowest band scores are within 1e-9 of each other
        sc = np.sort(det["scores"], axis=0)
        ties += int(np.sum((np.abs(sc[1] - sc[0]) <= 1e-9 * np.abs(sc[0])) & (sc[0] < A.MAXIMUM_VALUE)))
        checked += F
        wrf = A.stonemask(x, want, t, fs)
        assert np.array_equal(rf0[b, :F] > 0, wrf > 0)
        worst["stonemask"] = max(worst["stonemask"], float(np.max(np.abs(rf0[b, :F][v] / wrf[v] - 1), initial=0)))
        wsp = A.cheaptrick(x, rf0[b, :F], t, fs, n, stream)           # CheapTrick and sp2mc on the same f0
        worst["logsp"] = max(worst["logsp"], float(np.max(np.abs(np.log(sp[b, :F]) - np.log(wsp)))))
        wmc = A.sp2mc(wsp, 24, alpha)
        worst["mc"] = max(worst["mc"], float(np.max(np.abs(mc[b, :F] - wmc))))
    print("analysis fs=%d: worst %s; DIO score ties within 1e-9: %d of %d frames" % (fs, worst, ties, checked))
    assert worst["f0"] <= F0_TOL and worst["stonemask"] <= F0_TOL
    assert worst["logsp"] <= SP_TOL and worst["mc"] <= MC_TOL


def test_rows_are_bit_identical_at_any_position_and_padding(dev):
    fs = 16000
    rng = np.random.RandomState(3)
    waves = [wave(rng, fs, s)[0] for s in (2.2, 1.0, 3.1, 1.7)]
    full = run_chain(dev, waves, fs)
    for b, x in enumerate(waves):
        alone = run_chain(dev, [x], fs, pad=np.nan, S=len(x) + 777)
        other = run_chain(dev, [waves[(b + 1) % 4], x], fs, pad=12345.0)
        for k in range(1, 5):
            F = full[0][b]
            assert np.array_equal(alone[k][0, :F], full[k][b, :F]), (b, k)
            assert np.array_equal(other[k][1, :F], full[k][b, :F]), (b, k)


def test_status_word(dev):
    from gantts_b200 import ops
    fs = 16000
    rng = np.random.RandomState(4)
    x = wave(rng, fs, 1.0)[0]
    bad = x.copy()
    bad[100] = np.nan
    with pytest.raises(RuntimeError, match="not finite"):
        run_chain(dev, [x, bad], fs)
    with pytest.raises(RuntimeError, match="too short for DIO"):
        run_chain(dev, [x, x[:400]], fs)
    # padding beyond a row's length is never read
    assert run_chain(dev, [x[:8000]], fs, pad=np.nan)[0][0] == A.dio_frames(8000, fs, FP)
    # a StoneMask window over 4096 points: f0 = 41 Hz at 48 kHz
    xt = torch.from_numpy(np.stack([x, x])).to(dev)
    L = torch.tensor([len(x)] * 2, dtype=torch.int64, device=dev)
    f0, info = ops.world_dio(xt, L, 48000, FP)
    f0.fill_(41.0)
    ops.world_stonemask(xt, L, f0, info, 48000, FP)
    with pytest.raises(RuntimeError, match="over 4096"):
        ops.world_analysis_check(info)
    with pytest.raises(RuntimeError, match="fs = 1000"):
        ops.world_dio(xt, L, 1000, FP)


def test_smoothing_against_the_restatement(dev):
    from gantts_b200 import ops
    rng = np.random.RandomState(5)
    lens = [4096, 1, 300, 2500]
    x = np.full((4, 4096, 7), np.nan)
    for b, T in enumerate(lens):
        x[b, :T] = rng.randn(T, 7).cumsum(axis=0) * 0.1 + rng.randn(7)
    got = ops.modspec_smoothing(torch.from_numpy(x).to(dev), torch.tensor(lens, device=dev), 200.0).cpu().numpy()
    for b, T in enumerate(lens):
        want = A.modspec_smoothing(x[b, :T], 200.0)
        assert np.max(np.abs(got[b, :T] - want)) <= 1e-12 * max(1.0, np.max(np.abs(want)))
        assert np.all(got[b, T:] == 0)
    with pytest.raises(RuntimeError, match="at most n"):
        ops.modspec_smoothing(torch.zeros(1, 4097, 2, dtype=torch.float64, device=dev),
                              torch.tensor([5], device=dev), 200.0)


def test_synthesis_round_trip_recovers_f0(dev):
    """Analysing ops.world_synthesize output made from a known f0 and a smooth envelope: on frames voiced in both, five
    or more frames away from any V/UV change, the median error of the analysed f0 is under 0.5 % and 95 % of the frames
    are within 2 % of the synthesis f0 (the synthesis interpolates f0 between frames and adds aperiodic noise, so a
    frame's analysed f0 is not its own)."""
    from gantts_b200 import generate, ops
    fs = 16000
    rng = np.random.RandomState(6)
    n = generate.cheaptrick_fft_size(fs)
    F = 500
    t = np.arange(F)
    f0 = np.where((t // 90) % 2 == 0, 110 + 60 * np.sin(t / 40.0), 0.0)
    f0[:10] = 0
    mc = np.zeros((1, F, 25), np.float32)
    mc[0] = rng.randn(25) * np.exp(-0.4 * np.arange(25)) * 0.5
    mc[0, :, 0] += 4.0
    L = torch.tensor([F], dtype=torch.int64, device=dev)
    sp = ops.mc2sp(torch.from_numpy(mc).to(dev), L, generate.mcep_alpha(fs), n)
    ap = torch.full((1, F, n // 2 + 1), 0.001, dtype=torch.float64, device=dev)
    y, _ = ops.world_synthesize(torch.from_numpy(f0.astype(np.float32)[None]).to(dev), sp, ap, L, fs, FP)
    y = y.cpu().numpy()[0]
    frames, got, rf0 = run_chain(dev, [y], fs)[:3]
    m = min(F, int(frames[0]))
    voiced = (f0[:m] > 0) & (rf0[0, :m] > 0)
    steady = voiced.copy()
    for d in range(1, 6):
        steady[d:] &= f0[:m - d] > 0
        steady[:-d] &= f0[d:m] > 0
    err = np.abs(rf0[0, :m][steady] / f0[:m][steady] - 1)
    print("round trip: %d steady voiced frames, median |f0 error| %.2e, max %.2e" % (steady.sum(), np.median(err),
                                                                                    err.max()))
    assert steady.sum() > 100
    assert np.median(err) < 0.005 and np.mean(err < 0.02) >= 0.95


def test_command_with_and_without_wav_dir(dev, tmp_path, capsys):
    from scipy.io import wavfile
    from gantts_b200 import analysis, models, objective, train
    import train_cli_helpers as H
    root = str(tmp_path / "data")
    xd, yd = H.write_vc_data(root, n_files=16)
    hp = H.vc_hp()
    train.load_data(hp, xd, yd, -1)
    torch.manual_seed(3)
    model = getattr(models, hp.generator)(**hp.generator_params)
    ck = str(tmp_path / "ck" / "gan")
    os.makedirs(ck)
    train.save_checkpoint(model, torch.optim.Adagrad(model.parameters()), 4, ck, "Generator")
    ckpt = os.path.join(ck, "checkpoint_epoch4_Generator.pth")
    wd = str(tmp_path / "wavs")
    os.makedirs(wd)
    rng = np.random.RandomState(8)
    waves = {}
    for sub, xf, _ in objective.paired_files(xd, yd):
        for f in xf:
            name = os.path.splitext(os.path.basename(f))[0]
            waves[name] = wave(rng, 16000, rng.uniform(1.0, 2.0))[0].astype(np.int16)
            wavfile.write(os.path.join(wd, name + ".wav"), 16000, waves[name])
    base = ["--hparams_name=vc", xd, yd]
    assert objective.main(base + [str(tmp_path / "plain"), ckpt], hp=H.vc_hp()) == 0
    plain_out = capsys.readouterr().out
    for dst, extra in (("wav", []), ("wav1", ["--batch-size=1"])):
        assert objective.main(["--wav-dir=" + wd] + extra + base + [str(tmp_path / dst), ckpt], hp=H.vc_hp()) == 0
    printed = capsys.readouterr().out
    for sub, xf, _ in objective.paired_files(xd, yd):
        p, w, w1 = (np.load(str(tmp_path / d / (sub + ".npz"))) for d in ("plain", "wav", "wav1"))
        assert list(p["labels"]) == ["natural", "gan"] and "wav_lengths" not in p
        assert list(w["labels"]) == ["natural", "natural_wav", "gan"]
        for k in ("gv", "gv_mean", "ms_mean"):
            assert np.array_equal(w[k][[0, 2]], p[k]), k            # natural and the checkpoint: the same bits
            assert np.array_equal(w[k], w1[k]), k                   # any batch size: the same bits
        names = [os.path.splitext(os.path.basename(f))[0] for f in xf]
        assert list(w["wav_lengths"]) == [A.dio_frames(len(waves[nm]), 16000, FP) for nm in names]
        # natural_wav: the chain through analysis.analyse against the restatement, utterance by utterance
        for i, nm in enumerate(names[:3]):
            x = waves[nm].astype(np.float64)
            frames, _, rf0 = run_chain(dev, [x], 16000)[:3]
            t = np.arange(frames[0]) * FP / 1000.0
            sp = A.cheaptrick(x, rf0[0, :frames[0]], t, 16000)
            want = A.sp2mc(sp, hp.order, sptk_port.mcepalpha(16000))[:, 1:].astype(np.float32).astype(np.float64)
            assert np.all(np.abs(w["gv"][1, i] - np.var(want, axis=0)) <= 1e-5 * np.var(want, axis=0) + 1e-9)
        for ref in (0, 1):
            for label, g, m in objective.summary(list(w["labels"]), w["gv_mean"], w["ms_mean"], ref):
                line = ("%s %s: mean log10 GV ratio to %s %+.4f, RMS log MS difference to %s %.4f"
                        % (sub, label, w["labels"][ref], g, w["labels"][ref], m))
                assert line in printed
    assert "natural_wav" not in plain_out
    with pytest.raises(ValueError, match="kind must be"):
        analysis.analyse([np.zeros(100)], 16000, FP, 4, "tts_duration", dev)


def test_tts_chain_smooths_the_mel_cepstra(dev):
    from gantts_b200 import analysis
    fs = 16000
    rng = np.random.RandomState(9)
    waves = [wave(rng, fs, s)[0] for s in (1.3, 2.0)]
    mc, frames, _ = analysis.analyse(waves, fs, FP, 24, "tts_acoustic", dev)
    mc = mc.cpu().numpy()
    rf0 = run_chain(dev, waves, fs)[2]
    stream = A.randn_stream(int(frames.max()) * 2100)
    for b, x in enumerate(waves):
        t = np.arange(frames[b]) * FP / 1000.0
        sp = A.cheaptrick(x, rf0[b, :frames[b]], t, fs, 1024, stream)
        want = A.modspec_smoothing(A.sp2mc(sp, 24, sptk_port.mcepalpha(fs)), analysis.modulation_rate(fs, FP))
        assert mc.shape[2] == 25 and frames[b] == len(want)
        assert np.max(np.abs(mc[b, :frames[b]] - want)) <= MC_TOL
