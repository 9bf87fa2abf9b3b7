"""The Python-2 rewriting that tests/example_runner.py applies to the reference's example scripts (rbm_mnist.py, dbm_mnist.py)
so that they run unchanged against this package (north_star; SURVEY.md section 8 f.1)."""
from example_runner import translate


def test_translate_handles_the_two_python2_constructs_of_the_examples():
    src = 'print __doc__\ndef f((a, b), c,\n      (d, e), k=1):\n    print "x: {0}".format(a)\n    return a + e\n'
    g = {'__doc__': 'doc'}
    exec(compile(translate(src), '<t>', 'exec'), g)
    assert g['f']((1, 2), 3, (4, 5)) == 6
