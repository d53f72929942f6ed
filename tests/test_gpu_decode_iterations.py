"""The greedy decode kernel's iteration counter against the window structure recomputed on the host.  Every lock-step
iteration scores one window of up to 4 frames for each utterance with frames left and consumes it: blanks advance t, the
first emission ends the window, and reaching the symbol cap advances t.  So the number of iterations is the number of
windows of the utterance that needs the most, and it follows from the returned tokens, frames and counts alone."""
import pytest
import torch

pytestmark = pytest.mark.gpu

K_FRAMES = 4


def count_windows(frames, n_tok, T, max_symbols):
    """Windows consumed by an utterance of T valid encoder frames whose emissions happened at frames[:n_tok]."""
    t = sym = k = w = 0
    while t < T:
        w += 1
        for _ in range(min(K_FRAMES, T - t)):
            if k < n_tok and frames[k] == t:       # emits at frame t: the window ends here
                k += 1
                sym += 1
                if sym >= max_symbols:
                    t, sym = t + 1, 0
                break
            t, sym = t + 1, 0                        # blank
    assert k == n_tok, "every emission lies inside the utterance's frames"
    return w


@pytest.mark.parametrize("blank_bias", [None, -1e4], ids=["seeded", "symbol_cap"])
@pytest.mark.parametrize("B", [6, 37])
def test_decode_iterations_equal_the_longest_window_count(tiny_cfg, tiny_sd, B, blank_bias):
    from reazonspeech_b200.engine import Engine
    sd = dict(tiny_sd)
    if blank_bias is not None:
        b = sd["joint.joint_net.2.bias"].clone()
        b[tiny_cfg.blank] = blank_bias
        sd["joint.joint_net.2.bias"] = b
    eng = Engine(tiny_cfg, sd, "cuda:0")
    L = 48000
    g = torch.Generator().manual_seed(B)
    wav = 0.1 * torch.randn(B, L, generator=g)
    lens = torch.randint(L // 8, L + 1, (B,), generator=g, dtype=torch.int32)
    lens[0] = L
    lens[B - 1] = 1000                                 # one encoder frame
    U = eng.u_max(L)
    tokens, frames, n_tok = eng.transcribe_device(wav.cuda(), lens.cuda(), U)
    cycles = eng.decode_cycles(B, L, U)
    frames, n_tok = frames.cpu(), n_tok.cpu()
    T = [eng.lib.rs_enc_valid(eng.h, int(n)) for n in lens]
    w = [count_windows(frames[b].tolist(), int(n_tok[b]), T[b], tiny_cfg.max_symbols) for b in range(B)]
    print("tokens", n_tok.tolist()[:8], "frames", T[:8], "windows", w[:8])
    if blank_bias is not None:
        assert n_tok.tolist() == [t * tiny_cfg.max_symbols for t in T]
    assert cycles["iterations"] == max(1, max(w))
    for phase in ("phase_j", "barrier_a", "reduce", "phase_l", "barrier_b", "phase_p", "barrier_c", "j_loads", "j_rows", "j_misc"):
        assert cycles[phase] > 0, cycles
