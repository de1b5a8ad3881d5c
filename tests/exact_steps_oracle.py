"""TEST INFRASTRUCTURE ONLY: the Adam step from a dense fp64 gradient (gg_adam_apply_dense, DESIGN.md section 5.5) on
the host, in the kernel's operation order:

    g = f32(f64(scale * acc) + f64(f64(lam) * f64(x)))      fp64 mul, mul, add (numpy float64 does not contract)
    m, v, x: tests/update_bits_oracle.adam1 (the GG_ADAM1 sequence, all fp32)

lam is lam_emb for the rows and lam_bias for the biases.
"""
import numpy as np

from tests import update_bits_oracle as ubo

F = np.float32


def dense_g(acc, x, scale, lam):
    """the fp32 gradient of every element: one fp64 rounding per operation, then one to fp32"""
    acc = np.asarray(acc, np.float64)
    x = np.asarray(x, F).astype(np.float64)
    return (np.float64(scale) * acc + np.float64(F(lam)) * x).astype(F)


def dense_step(state, acc_emb, acc_bias, scale, lam_emb, lam_bias, lt, b1=0.9, b2=0.999, eps=1e-8):
    """One step in place on state = {emb, m_emb, v_emb, bias_t, m_bias, v_bias} (fp32 numpy, emb padded)."""
    b1, b2, eps = F(b1), F(b2), F(eps)
    g = dense_g(acc_emb, state["emb"], scale, lam_emb)
    gb = dense_g(acc_bias, state["bias_t"], scale, lam_bias)
    ubo.adam1(state["emb"], state["m_emb"], state["v_emb"], g, lt, b1, b2, eps)
    ubo.adam1(state["bias_t"], state["m_bias"], state["v_bias"], gb, lt, b1, b2, eps)


def dense_step_literal(state, acc_emb, acc_bias, scale, lam_emb, lam_bias, lt, b1=0.9, b2=0.999, eps=1e-8):
    """The same step as a literal loop of numpy scalars, element by element (the statement ``dense_step`` must equal)."""
    b1, b2, eps, lt = F(b1), F(b2), F(eps), F(lt)
    omb1, omb2 = F(F(1) - b1), F(F(1) - b2)

    def one(x, m, v, a, lam):
        g = F(np.float64(np.float64(scale) * np.float64(a)) + np.float64(np.float64(F(lam)) * np.float64(x)))
        m = F(F(m * b1) + F(omb1 * g))
        v = F(F(v * b2) + F(F(g * g) * omb2))
        x = F(x - F(F(lt * m) / F(F(np.sqrt(v)) + eps)))
        return x, m, v
    E, mE, vE = state["emb"], state["m_emb"], state["v_emb"]
    for r in range(E.shape[0]):
        for c in range(E.shape[1]):
            E[r, c], mE[r, c], vE[r, c] = one(E[r, c], mE[r, c], vE[r, c], acc_emb[r, c], lam_emb)
        state["bias_t"][r], state["m_bias"][r], state["v_bias"][r] = one(state["bias_t"][r], state["m_bias"][r],
                                                                       state["v_bias"][r], acc_bias[r], lam_bias)


def random_state(n, n_emb, ld, rs):
    """padded parameters and a nonzero Adam state (m of both signs, v >= 0), pad columns 0"""
    st = {}
    for k, s in (("emb", 0.5), ("m_emb", 1e-3), ("v_emb", 1e-6)):
        a = np.zeros((n, ld), F)
        a[:, :n_emb] = rs.normal(0, s, (n, n_emb)).astype(F)
        st[k] = np.abs(a) if k == "v_emb" else a
    st["bias_t"] = rs.normal(0, 0.3, n).astype(F)
    st["m_bias"] = rs.normal(0, 1e-3, n).astype(F)
    st["v_bias"] = np.abs(rs.normal(0, 1e-6, n)).astype(F)
    return st
