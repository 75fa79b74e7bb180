"""Every disentanglement score of `disvae.evaluate.SCORES` in training, in a sweep and across a resume, on the GPU:
turning a score on leaves training, MIG / AAM and the other scores bit-identical, and writes each epoch's score as a
standalone Evaluator does under the documented seed; a sweep member's scores, during training and from
`Sweep.evaluate`, equal its lone run's; a resumed run writes the same later scores as the run that was never stopped.

Run as a script (`python tests/test_scores_gpu.py FLAG PHASE SAVE_DIR OUT`) it trains the resume case's stopped
("first") or continued ("resume") run of the score whose flag is FLAG in a fresh process and saves its result to OUT.
"""
import os
import subprocess
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if __name__ == "__main__":                 # a resume phase in a fresh process: the paths conftest.py gives the tests
    sys.path[:0] = [os.path.join(ROOT, "disentangling-vae_b200"), HERE]

from disvae.evaluate import SCORES, epoch_metrics_filenames, epoch_score_filenames, evaluation_seed  # noqa: E402
from test_eval_resident_gpu import (EPOCHS, IMG, K, _assert_same_eval_files, _assert_same_state, _dataset,  # noqa: E402
                                    _evaluator, _loader, _loss, _member, _n_samples, _state)

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SPECS = [("btcvae", 11), ("betaB", 12), ("factor", 13)]
RESUME_LOSS = {"factor_score": "factor", "sap_score": "btcvae", "beta_vae_score": "btcvae"}
each_score = pytest.mark.parametrize("score", SCORES, ids=[s.flag for s in SCORES])


def _eval_args(score, seed):
    """The Evaluator's keywords for `score` alone."""
    return {"is_" + score.flag: True, score.flag + "_seed": seed}


def _files(score):
    return [(score.filename,) * 2, (score.helpers_file,) * 2]


def _epoch_files(scores, epochs=EPOCHS):
    """(name, name) of the MIG / AAM files and the files of `scores` of every epoch."""
    names = [n for e in range(epochs) for n in epoch_metrics_filenames(e)]
    names += [n for e in range(epochs) for s in scores for n in epoch_score_filenames(s, e)]
    return [(n, n) for n in names]


def _standalone_score(score, kind, save_dir, epoch, noise_key, out_dir):
    """The documented reproduction of the score's files of epoch `epoch`: model-{epoch}.pt in a fresh model, an
    Evaluator over DataLoader(dataset, 1000, shuffle=False) with seed evaluation_seed(noise key, epoch)."""
    import disvae
    from synthetic_factors import loader
    m = disvae.init_specific_model("Burgess", IMG, 10)
    m.load_state_dict(torch.load(os.path.join(save_dir, "model-%d.pt" % epoch), weights_only=True))
    _evaluator(m.to(DEV), _loss(kind, K ** 4), out_dir)(loader(_dataset(), 1000), is_metrics=False, is_losses=False,
                                                        **_eval_args(score, evaluation_seed(noise_key, epoch)))


@each_score
def test_score_leaves_training_unchanged(tmp_path, score):
    """Both runs write every other score; the second writes this one too."""
    seed = 17
    others = [s for s in SCORES if s is not score]
    runs = {}
    with _n_samples(512):
        for on in (False, True):
            tr = _member("btcvae", seed, tmp_path / ("on%d" % on))
            torch.manual_seed(seed)
            tr(_loader(), epochs=EPOCHS, checkpoint_every=1, metrics_every=1,
               **{s.flag: True for s in SCORES if on or s is not score})
            runs[on] = tr
    _assert_same_state(_state(runs[True]), _state(runs[False]), "%s on vs off" % score.flag)
    _assert_same_eval_files(runs[True].save_dir, runs[False].save_dir,
                            _epoch_files(others) + [("train_losses.log",) * 2], "the other files with and without the score",
                            nan_equal=True)
    assert not any(f.startswith(score.stem) for f in os.listdir(runs[False].save_dir))
    key = runs[True].training_state()["noise"]["key"]
    for e in range(EPOCHS):
        out = tmp_path / ("standalone%d" % e)
        _standalone_score(score, "btcvae", runs[True].save_dir, e, key, out)
        pairs = list(zip(epoch_score_filenames(score, e), (score.filename, score.helpers_file)))
        _assert_same_eval_files(runs[True].save_dir, out, pairs, e, nan_equal=True)


@each_score
def test_sweep_scores_equal_lone_runs(tmp_path, score):
    from disvae.sweep import Sweep
    from synthetic_factors import loader
    with _n_samples(512):
        members = [_member(kind, seed, tmp_path / ("m%d_%s" % (k, kind))) for k, (kind, seed) in enumerate(SPECS)]
        sweep = Sweep(members, seeds=[seed for _, seed in SPECS])
        sweep(_loader(), epochs=EPOCHS, checkpoint_every=1, metrics_every=1, **{score.flag: True})
        sweep.evaluate(is_metrics=False, is_losses=False, **{"is_" + score.flag: True})
        lones = []
        for kind, seed in SPECS:
            tr = _member(kind, seed, tmp_path / ("lone_" + kind))
            torch.manual_seed(seed)
            tr(_loader(), epochs=EPOCHS, checkpoint_every=1, metrics_every=1, **{score.flag: True})
            _evaluator(tr.model, tr.loss_f, tr.save_dir)(loader(_dataset(), 1000), is_losses=False,
                                                         **_eval_args(score, evaluation_seed(seed, EPOCHS - 1)))
            lones.append(tr)
    for m, lone, (kind, _) in zip(members, lones, SPECS):
        _assert_same_state(_state(m), _state(lone), kind)
        _assert_same_eval_files(m.save_dir, lone.save_dir, _epoch_files([score]) + _files(score), kind, nan_equal=True)
        last = list(zip((score.filename, score.helpers_file), epoch_score_filenames(score, EPOCHS - 1)))
        _assert_same_eval_files(m.save_dir, m.save_dir, last, kind, nan_equal=True)


def _resume_run(score, phase, save_dir):
    """'full': EPOCHS epochs; 'first': 1 epoch; 'resume': load training-state-0.pt and train EPOCHS - 1 more.  All with
    save_state=True, metrics_every=1 and the score on."""
    from disvae.utils.modelIO import load_training_state
    tr = _member(RESUME_LOSS[score.flag], 29, save_dir)
    if phase == "resume":
        load_training_state(tr, os.path.join(str(save_dir), "training-state-0.pt"))
    torch.manual_seed(29)
    epochs = {"full": EPOCHS, "first": 1, "resume": EPOCHS - 1}[phase]
    with _n_samples(512):
        tr(_loader(), epochs=epochs, checkpoint_every=1, save_state=True, metrics_every=1, **{score.flag: True})
    torch.cuda.synchronize()
    return _state(tr)


@each_score
def test_resumed_run_writes_the_same_later_scores(tmp_path, score):
    full = _resume_run(score, "full", tmp_path / "a")
    for phase in ("first", "resume"):
        r = subprocess.run([sys.executable, os.path.abspath(__file__), score.flag, phase, str(tmp_path / "b"),
                            str(tmp_path / (phase + ".pt"))], capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, (phase, r.stdout[-2000:] + r.stderr[-4000:])
    got = torch.load(tmp_path / "resume.pt", weights_only=False)
    _assert_same_state(got, full, "resumed")
    _assert_same_eval_files(tmp_path / "b", tmp_path / "a", _epoch_files([score]), "resume", nan_equal=True)


if __name__ == "__main__":
    flag, phase, save_dir, out = sys.argv[1:5]
    torch.cuda.set_device(DEV)
    torch.save(_resume_run(next(s for s in SCORES if s.flag == flag), phase, save_dir), out)
