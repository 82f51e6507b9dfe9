"""The plugin registry of the replay path and the drop-in switch.

`agents`, `retrieve_methods`, `update_methods` mirror the dicts of the reference's
utils/name_match.py:31-55 for the entries on the replay path.  `install()` mutates the
reference's own dicts in place (the objects `experiment/run.py:5` and `utils/buffer/buffer.py:2`
already hold), so `general_main.py` runs unchanged:

    import b200ocl; b200ocl.install()          # before main(args); or:  python -m b200ocl.launch general_main.py ...

The agents registered here are ER, SCR, AGEM, LWF, ICARL and GDUMB.  `extra_agents` holds agents that are only
registered on request, `install(extra=('EWC',))` (or `B200OCL_EXTRA_AGENTS=EWC` with b200ocl.launch): EWC (EWC++).
Every other agent / plugin of the reference (EWC unless requested, CNDPM, the match retrievals) stays registered and
untouched.

With B200OCL_CONCURRENT_RUNS=R (an integer > 1) install() also replaces experiment.run.multiple_run with
multirun.multiple_run, which trains R repetitions of the experiment at once (general_main.py and main_config.py import it
by name after install()), and, when experiment.run defines it, experiment.run.multiple_run_tune_separate with
multirun.multiple_run_tune_separate, which trains R of main_tune.py's tuning and final trainings at once (main_tune.py
imports it by name after install()).  uninstall() puts both back; an attribute experiment.run lacked stays absent.  Unset
or 1 leaves them alone; any other value, and every refusal of multirun.check_concurrent, raises ValueError before
anything is replaced.

With B200OCL_RUN_DEVICES (a comma-separated list of CUDA ordinals, e.g. 0,1,2,3 or 0,0) install() replaces the same
two drivers whatever R is: their trainings then run in worker processes, one per list entry, R at a time in each.  A
non-integer, a negative ordinal or an empty entry raises ValueError, as do the refusals of R > 1.  Unset or empty
changes nothing.

With B200OCL_CHECKPOINT_DIR (a directory) install() replaces the same two drivers whatever R is, so that an
interrupted experiment resumes from its last finished task (checkpoint.py).  Parity mode and data-parallel gradient sync
are refused with ValueError before anything is replaced.  Unset or empty changes nothing.

With B200OCL_CHECKPOINT_ASYNC=1 as well, the snapshots are staged on the device and written behind the runs
(checkpoint.py).  Unset, empty or 0 changes nothing; any other value, or 1 without a checkpoint directory, raises
ValueError in install() before anything is replaced.
"""
from .learners import AGEM, EWC_pp, ExperienceReplay, Gdumb, Icarl, Lwf, SupContrastReplay
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

# opt-in: install(extra=...) replaces these entries only when named
extra_agents = {
    'EWC': EWC_pp,
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
installed_extra = ()      # the extra agents of the last install(); worker processes install the same


def install(reference_name_match=None, extra=()):
    """Swap the replay-path entries of the reference registries for the CUDA-backed classes, and the agents of
    extra_agents named in `extra`.  Returns the dict of what was replaced (also kept for uninstall())."""
    import importlib
    extra = tuple(extra)
    unknown = [k for k in extra if k not in extra_agents]
    if unknown:
        raise ValueError('unknown extra agent(s) %s; available: %s' % (', '.join(map(repr, unknown)),
                                                                      ', '.join(sorted(extra_agents))))
    from . import checkpoint, multirun
    n_concurrent = multirun.concurrent_runs()
    devices = multirun.run_devices()
    multirun.check_concurrent(n_concurrent, devices=devices)
    directory = checkpoint.checkpoint_dir()
    checkpoint.check_checkpoint(directory)
    checkpoint.checkpoint_async()
    if reference_name_match is None:
        reference_name_match = importlib.import_module('utils.name_match')
    nm = reference_name_match
    replaced = {}
    chosen = dict(agents, **{k: extra_agents[k] for k in extra})
    for table_name, mine in (('agents', chosen), ('retrieve_methods', retrieve_methods),
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
    if n_concurrent > 1 or devices or directory:
        run = importlib.import_module('experiment.run')
        replaced[('experiment.run', 'multiple_run')] = run.multiple_run
        run.multiple_run = multirun.multiple_run
        if hasattr(run, 'multiple_run_tune_separate'):     # a reference without main_tune.py's loop keeps none
            replaced[('experiment.run', 'multiple_run_tune_separate')] = run.multiple_run_tune_separate
            run.multiple_run_tune_separate = multirun.multiple_run_tune_separate
    _installed.update(replaced)
    global installed_extra
    installed_extra = extra
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
    global installed_extra
    installed_extra = ()
