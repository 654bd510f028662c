#!/usr/bin/env python
"""Records tests/golden/spec_text_answers.json: what oracle/tla_eval.py answers, run on the TEXT of the reference's
vsr-revisited/paper/VSR.tla, to the questions tests/test_spec_text.py asks — successor multisets (as hashes), invariant
verdicts, level sizes, orbit counts — in the order it asks them.  The tests replay these answers wherever the spec's
text is absent.  Run it where a checkout of the reference (Vanlightly/vsr-tlaplus) is at hand; it runs the tests once
against the text:

    python tests/golden/make_spec_text_answers.py <reference checkout>
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    spec = os.path.join(os.path.abspath(sys.argv[1]), "vsr-revisited", "paper", "VSR.tla")
    if not os.path.exists(spec):
        sys.exit("no %s" % spec)
    env = dict(os.environ, VSR_SPEC_TLA=spec)
    sys.exit(subprocess.call([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.join(ROOT, "tests", "test_spec_text.py")],
                             env=env, cwd=ROOT))


if __name__ == "__main__":
    main()
