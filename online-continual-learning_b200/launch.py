"""Run the reference's unchanged entry point with the replay path switched to the CUDA engine:

    python -m b200ocl.launch /path/to/reference/general_main.py --agent ER --retrieve ASER --update ASER ...

The reference tree is put first on sys.path, its registries are patched in place
(b200ocl.registry.install) and general_main.py is executed with runpy, byte-identical.  Any entry point of the reference
runs the same way, main_tune.py included.
B200OCL_EXTRA_AGENTS (comma-separated, e.g. EWC or EWC,DERPP,PCR,GEM) also registers those opt-in agents (registry.extra_agents)."""
import os
import runpy
import sys


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv:
        raise SystemExit('usage: python -m b200ocl.launch <reference>/general_main.py [reference args...]')
    script = os.path.abspath(argv[0])
    sys.path.insert(0, os.path.dirname(script))
    from b200ocl import registry
    extra = [k.strip() for k in os.environ.get('B200OCL_EXTRA_AGENTS', '').split(',') if k.strip()]
    registry.install(extra=extra)
    sys.argv = [script] + argv[1:]
    runpy.run_path(script, run_name='__main__')


if __name__ == '__main__':
    main()
