"""build() copies the unmodified reference (lschoe/mpyc: `mpyc/`, `demos/`, `tests/`) from $MPYC_REFERENCE or
DEFAULT_SRC to the git-ignored oracle/_ref/, for the tests that run its own runtime, tests and demos on the engine and
for `bench.py --impl reference`; the copy travels with the built tree.  Without it those tests skip."""
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
DEST = os.path.join(HERE, '_ref')
DEFAULT_SRC = '/root/reference'   # where build hosts keep the read-only reference checkout
PARTS = ('mpyc', 'demos', 'tests')


def _is_reference(path):
    return bool(path) and os.path.isfile(os.path.join(path, 'mpyc', 'thresha.py'))


def install(src=None):
    """Copy the reference checkout `src` (default $MPYC_REFERENCE, else DEFAULT_SRC) to oracle/_ref/; returns its path,
    or None when there is no checkout to copy."""
    src = src or os.environ.get('MPYC_REFERENCE') or DEFAULT_SRC
    if not _is_reference(src):
        return None
    if os.path.realpath(src) == os.path.realpath(DEST):
        return DEST
    tmp = DEST + '.tmp'
    shutil.rmtree(tmp, ignore_errors=True)
    os.makedirs(tmp)
    for part in PARTS:
        if os.path.isdir(os.path.join(src, part)):
            shutil.copytree(os.path.join(src, part), os.path.join(tmp, part), copy_function=shutil.copyfile,
                            ignore=shutil.ignore_patterns('__pycache__', '*.pyc'))
    for root, _, _ in os.walk(tmp):   # copytree gives directories the checkout's (read-only) modes: keep the copy removable
        os.chmod(root, 0o755)
    shutil.rmtree(DEST, ignore_errors=True)
    os.rename(tmp, DEST)
    return DEST


def path():
    """Directory holding the reference's `mpyc` package: $MPYC_REFERENCE, else oracle/_ref/, else None."""
    for cand in (os.environ.get('MPYC_REFERENCE'), DEST):
        if _is_reference(cand):
            return cand
    return None
