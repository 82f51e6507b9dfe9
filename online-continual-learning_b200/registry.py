"""The plugin registry of the replay path and the drop-in switch.

`agents`, `retrieve_methods`, `update_methods` mirror the dicts of the reference's
utils/name_match.py:31-55 for the entries on the replay path.  `install()` mutates the
reference's own dicts in place (the objects `experiment/run.py:5` and `utils/buffer/buffer.py:2`
already hold), so `general_main.py` runs unchanged:

    import b200ocl; b200ocl.install()          # before main(args); or:  python -m b200ocl.launch general_main.py ...

The agents registered here are ER, SCR, AGEM, LWF, ICARL and GDUMB.  Every other agent / plugin of the reference
(EWC, CNDPM, the match retrievals) stays registered and untouched.
"""
from .learners import AGEM, ExperienceReplay, Gdumb, Icarl, Lwf, SupContrastReplay
from .retrieve import ASER_retrieve, MIR_retrieve, Random_retrieve
from .update import ASER_update, GSSGreedyUpdate, Reservoir_update

agents = {
    'ER': ExperienceReplay,
    'SCR': SupContrastReplay,
    'AGEM': AGEM,
    'LWF': Lwf,
    'ICARL': Icarl,
    'GDUMB': Gdumb,
}

retrieve_methods = {
    'MIR': MIR_retrieve,
    'random': Random_retrieve,
    'ASER': ASER_retrieve,
}

update_methods = {
    'random': Reservoir_update,
    'GSS': GSSGreedyUpdate,
    'ASER': ASER_update,
}

_installed = {}


def install(reference_name_match=None):
    """Swap the replay-path entries of the reference registries for the CUDA-backed classes.
    Returns the dict of what was replaced (also kept for uninstall())."""
    import importlib
    if reference_name_match is None:
        reference_name_match = importlib.import_module('utils.name_match')
    nm = reference_name_match
    replaced = {}
    for table_name, mine in (('agents', agents), ('retrieve_methods', retrieve_methods),
                             ('update_methods', update_methods)):
        table = getattr(nm, table_name)
        for key, cls in mine.items():
            replaced[(table_name, key)] = table.get(key)
            table[key] = cls                      # in place: run.py / buffer.py hold the same dict objects
    # name-bound imports that are resolved at their use site (SURVEY.md section 8b)
    from .losses import SupConLoss
    from .shapley import compute_knn_sv
    patches = [('agents.base', 'SupConLoss', SupConLoss),
               ('utils.buffer.aser_retrieve', 'compute_knn_sv', compute_knn_sv),
               ('utils.buffer.aser_update', 'compute_knn_sv', compute_knn_sv)]
    for mod_name, attr, obj in patches:
        try:
            mod = importlib.import_module(mod_name)
        except ImportError:
            continue
        replaced[(mod_name, attr)] = getattr(mod, attr, None)
        setattr(mod, attr, obj)
    _installed.update(replaced)
    return replaced


def uninstall(reference_name_match=None):
    import importlib
    if reference_name_match is None:
        reference_name_match = importlib.import_module('utils.name_match')
    for (where, key), old in list(_installed.items()):
        if where in ('agents', 'retrieve_methods', 'update_methods'):
            table = getattr(reference_name_match, where)
            if old is None:
                table.pop(key, None)
            else:
                table[key] = old
        elif old is not None:
            setattr(importlib.import_module(where), key, old)
    _installed.clear()
