"""Checkpoint IO with the reference's on-disk format (disvae/utils/modelIO.py:14-173):
`model.pt` is a plain state_dict with the reference's keys, `specs.json` the metadata, so
checkpoints shipped with the reference (results/*/model.pt) load into this implementation.  `training-state-*.pt`
files (save_training_state) hold what continuing a run needs besides the weights."""
import json
import os
import re

import numpy as np
import torch

MODEL_FILENAME = "model.pt"
META_FILENAME = "specs.json"
TRAINING_STATE_PREFIX = "training-state-"


def save_metadata(metadata, directory, filename=META_FILENAME, **kwargs):
    with open(os.path.join(directory, filename), "w") as f:
        json.dump(metadata, f, indent=4, sort_keys=True, **kwargs)


def load_metadata(directory, filename=META_FILENAME):
    with open(os.path.join(directory, filename)) as f:
        return json.load(f)


def save_model(model, directory, metadata=None, filename=MODEL_FILENAME):
    """modelIO.py:14-42: state_dict saved from CPU copies; the model stays on its device."""
    if metadata is None:
        metadata = dict(img_size=model.img_size, latent_dim=model.latent_dim, model_type=model.model_type)
    save_metadata(metadata, directory)
    state = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    torch.save(state, os.path.join(directory, filename))


def load_model(directory, is_gpu=True, filename=MODEL_FILENAME):
    """modelIO.py:81-104"""
    from disvae.models.vae import init_specific_model
    device = torch.device("cuda" if torch.cuda.is_available() and is_gpu else "cpu")
    meta = load_metadata(directory)
    model = init_specific_model(meta["model_type"], meta["img_size"], meta["latent_dim"]).to(device)
    model.load_state_dict(torch.load(os.path.join(directory, filename), map_location=device), strict=False)
    model.eval()
    return model


def load_checkpoints(directory, is_gpu=True):
    """modelIO.py:107-127"""
    checkpoints = []
    for root, _, filenames in os.walk(directory):
        for filename in filenames:
            if filename.startswith(TRAINING_STATE_PREFIX):          # not a model checkpoint
                continue
            results = re.search(r'.*?-([0-9].*?).pt', filename)
            if results is not None:
                checkpoints.append((int(results.group(1)), load_model(root, is_gpu=is_gpu, filename=filename)))
    return checkpoints


def save_training_state(trainer, directory, filename):
    """`trainer.training_state()` (disvae.training.Trainer) saved to directory/filename; returns the path."""
    path = os.path.join(directory, filename)
    torch.save(trainer.training_state(), path)
    return path


def load_training_state(trainer, path):
    """Apply the training state saved at `path` to `trainer` (Trainer.load_training_state); returns the state."""
    state = torch.load(path, map_location="cpu", weights_only=True)
    trainer.load_training_state(state)
    return state


def numpy_serialize(obj):
    if type(obj).__module__ == np.__name__:
        return obj.tolist() if isinstance(obj, np.ndarray) else obj.item()
    raise TypeError('Unknown type:', type(obj))


def save_np_arrays(arrays, directory, filename):
    save_metadata(arrays, directory, filename=filename, default=numpy_serialize)


def load_np_arrays(directory, filename):
    return {k: np.array(v) for k, v in load_metadata(directory, filename=filename).items()}
