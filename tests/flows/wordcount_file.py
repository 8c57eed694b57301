"""Config C0 (BASELINE.json configs[0]) written against `bytewax` (load it with compat/ on PYTHONPATH): the reference's
examples/wordcount.py pipeline -- file lines -> lower case -> tokens -> count_final -> stdout -- over its sample text,
stored as tests/golden/wordcount.txt.  Run from the repository root."""
import re

import bytewax.operators as op
from bytewax.connectors.files import FileSource
from bytewax.connectors.stdio import StdOutSink
from bytewax.dataflow import Dataflow

flow = Dataflow("wordcount")
lines = op.input("inp", flow, FileSource("tests/golden/wordcount.txt"))
lower = op.map("lower", lines, str.lower)
tokens = op.flat_map("tokenize", lower, lambda line: re.findall(r'[^\s!,.?":;0-9]+', line))
counts = op.count_final("count", tokens, lambda word: word)
op.output("out", counts, StdOutSink())
