import pytest

# shared check bodies outside the test modules keep pytest's detailed assertion messages
pytest.register_assert_rewrite("tests.step_cases", "tests.golden_inputs", "tests.transcode_cases")
