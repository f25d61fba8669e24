"""CPU: the builders build what the reference's own builders build.

tests/golden/reference_builders.json records the graphs the reference's five builder SOURCE FILES build when
they are executed unmodified on this package (tests/golden/generate_builders.py): inputs, layer sequence
(class + Keras-style name), weights (name + shape + trainable), planner slots (i.e. the same single fused
gather launch), and every builder keyword with its default.  deepctr_b200.models must build the same graphs
for the same columns (model_golden_checks, shared by every fixture family).  Graph construction needs no GPU.
"""
import model_golden_checks as C

T = C.model_tests("models")
test_reference_builder_source_runs_on_this_package = T.graph
test_reference_default_arguments_are_the_same = T.defaults
