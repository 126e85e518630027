"""Config loading with the reference's semantics (src/config.py:10-59): `inherit_from` is read recursively, a file without it falls back
to `default_path`, and update_recursive merges -- a nested dict merges into what is below it, anything else replaces it.  Paths are
opened as given, relative to the current directory, as the reference (run from its repository root) opens them."""
import yaml


def load_config(path, default_path=None):
    """The merged config dict of the yaml file `path`."""
    with open(path, "r") as f:
        cfg_special = yaml.full_load(f)
    inherit_from = cfg_special.get("inherit_from")
    if inherit_from is not None:
        cfg = load_config(inherit_from, default_path)
    elif default_path is not None:
        with open(default_path, "r") as f:
            cfg = yaml.full_load(f)
    else:
        cfg = dict()
    update_recursive(cfg, cfg_special)
    return cfg


def update_recursive(dict1, dict2):
    """Merge dict2 into dict1 in place: a dict value merges into dict1's entry (a scalar there is replaced by a dict first), any other
    value replaces it.  A dict over a scalar replaces the scalar with the dict (the reference raises there)."""
    for k, v in dict2.items():
        if k not in dict1:
            dict1[k] = dict()
        if isinstance(v, dict):
            if not isinstance(dict1[k], dict):
                dict1[k] = dict()
            update_recursive(dict1[k], v)
        else:
            dict1[k] = v
