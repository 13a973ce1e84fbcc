#!/usr/bin/env python
"""Generate tests/golden/index_goldens.json from the reference tree.

Run where the reference tree is (see make_golden.py); the output travels with
the repo.  It holds every "# dn query ..." section of the reference's
`dn build` + `dn query` goldens, split as make_golden.py splits the scan
goldens ({cmd, argv, header, text}):

  tests/dn/local/tst.index_file.sh.out
  tests/dn/local/tst.index_fileset.sh.out

plus, under "find", the lines before each file's first section: for the
fileset test, the listing of the index files its hourly build creates.

These are the reference's test vectors, not its source.
"""

import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import HERE, REF, parse_argv, split_sections  # noqa: E402


def main():
    out = {'suites': {}, 'find': {}}
    for suite, path in [
            ('index_file', 'tests/dn/local/tst.index_file.sh.out'),
            ('index_fileset', 'tests/dn/local/tst.index_fileset.sh.out')]:
        text = open(os.path.join(REF, path)).read()
        secs = []
        for s in split_sections(text):
            cmd, argv = parse_argv(s['header'])
            secs.append({'cmd': cmd, 'argv': argv, 'header': s['header'],
                         'text': '\n'.join(s['lines'])})
        out['suites'][suite] = secs
        out['find'][suite] = text[:text.find('# dn ')].split('\n')[:-1]
    with open(os.path.join(HERE, 'index_goldens.json'), 'w') as f:
        json.dump(out, f, indent=0, sort_keys=True)
    print('wrote', sum(len(v) for v in out['suites'].values()),
          'query sections')


if __name__ == '__main__':
    sys.exit(main())
