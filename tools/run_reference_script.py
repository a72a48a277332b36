"""Run one of the reference's own task scripts, byte-identical, on this package:

    python tools/run_reference_script.py /path/to/ClipBERT src/tasks/run_video_retrieval.py --config ... [script args]
    python -m torch.distributed.run --nproc-per-node 8 tools/run_reference_script.py /path/to/ClipBERT src/tasks/run_video_retrieval.py ...

It (1) registers stand-ins for `horovod.torch` and `apex` when they are not installed (clipbert_b200.compat.install),
(2) aliases `src.modeling.{e2e_model,modeling,grid_feat}` to the H100 modules (compat.alias_reference_modules) so that the
script's own `from src.modeling.e2e_model import ClipBert` lines import them, (3) runs the script as `__main__` from the
reference root. Everything else the script imports (easydict, tensorboardX, ujson, av, lmdb: data loading and logging) must be
installed - those sit outside the hot path this package replaces.
"""
import os
import runpy
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    if len(sys.argv) < 3:
        sys.exit(__doc__)
    ref_root, script = os.path.abspath(sys.argv[1]), sys.argv[2]
    sys.path.insert(0, ROOT)
    sys.path.insert(0, ref_root)
    import clipbert_b200.compat as compat
    print("[clipbert_b200] stand-ins registered: %s; aliased: %s" % (compat.install(), compat.alias_reference_modules()), file=sys.stderr)
    os.chdir(ref_root)
    sys.argv = [script] + sys.argv[3:]
    runpy.run_path(os.path.join(ref_root, script), run_name="__main__")


if __name__ == "__main__":
    main()
