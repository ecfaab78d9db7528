"""GMF / WRMF(embedding_dtype=...): the keyword is checked before any table is made, so this runs without a GPU."""
import pytest

from openrec_b200.tf2.recommenders import GMF, WRMF


@pytest.mark.parametrize("cls", (GMF, WRMF))
@pytest.mark.parametrize("dtype", ("float16", "bf16", "float64", None))
def test_unknown_embedding_dtype_refused(cls, dtype):
    with pytest.raises(ValueError, match="embedding_dtype"):
        cls(8, 8, 10, 20, embedding_dtype=dtype)
