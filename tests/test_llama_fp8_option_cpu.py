"""`llama_ffn` reads its fp8 option (argument or TUTEL_B200_FP8) with the values `ffn` accepts, and refuses MX."""
import pytest


def _llama(fp8=None):
    from tutel_b200.models.experts.llama_ffn import LlamaFFNNetwork
    return LlamaFFNNetwork(32, 64, 2, 1, fp8=fp8)


@pytest.mark.parametrize('value,on', [('1', True), ('true', True), ('TRUE', True), ('row', True), ('0', False),
                                      ('false', False), ('none', False)])
def test_llama_fp8_environment_values(monkeypatch, value, on):
    monkeypatch.setenv('TUTEL_B200_FP8', value)
    assert _llama().fp8 is on


@pytest.mark.parametrize('value,on', [(True, True), (False, False), ('row', True), (1, True), (0, False)])
def test_llama_fp8_argument_values(monkeypatch, value, on):
    monkeypatch.setenv('TUTEL_B200_FP8', '1')            # an explicit argument wins over the environment
    assert _llama(value).fp8 is on


def test_llama_fp8_rejects_mx(monkeypatch):
    with pytest.raises(AssertionError, match='mx'):
        _llama('mx')
    monkeypatch.setenv('TUTEL_B200_FP8', 'mx')
    with pytest.raises(AssertionError, match='"row"'):
        _llama()
