"""Drop-in alias: `import uisrnn` gives the public surface of google/uis-rnn
(its `uisrnn/__init__.py:21-30`) backed by the H100-native package `uisrnn_b200`.
Sub-modules (`uisrnn.uisrnn`, `uisrnn.utils`, `uisrnn.evals`, `uisrnn.loss_func`,
`uisrnn.arguments`, `uisrnn.contrib.*`) resolve to the same module objects."""
import sys as _sys

from uisrnn_b200 import arguments, contrib, evals, loss_func, uisrnn, utils  # noqa: F401
from uisrnn_b200.contrib import contrib_template, range_search_crp_alpha

for _name, _module in (('arguments', arguments), ('contrib', contrib), ('evals', evals),
                       ('loss_func', loss_func), ('uisrnn', uisrnn), ('utils', utils),
                       ('contrib.contrib_template', contrib_template),
                       ('contrib.range_search_crp_alpha', range_search_crp_alpha)):
  _sys.modules[__name__ + '.' + _name] = _module

parse_arguments = arguments.parse_arguments
compute_sequence_match_accuracy = evals.compute_sequence_match_accuracy
output_result = utils.output_result
UISRNN = uisrnn.UISRNN
parallel_predict = uisrnn.parallel_predict
