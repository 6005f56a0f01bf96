"""Stand-in for lightning (absent offline) so that the reference's EvaluationIndexGenerator imports and its
test_step runs on the CPU outside a Trainer; see lightning/pytorch."""
