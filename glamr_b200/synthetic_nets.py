"""Seeded stand-in weights for the learned prior (no pretrained checkpoints exist offline).

``infiller_param_shapes()`` / ``trajpred_param_shapes()`` list every inference-path parameter under its reference
state-dict name (motion_infiller/models/motion_infiller_vae.py, traj_pred/models/traj_pred_vae.py with the shipped
configs); ``make_state(shapes, seed)`` fills them deterministically (numpy), so the reference (golden generation),
the oracle and the CUDA library all run the very same network.
"""
import numpy as np

D, NZ, FF = 256, 128, 512


def _attn(prefix):
    return {f'{prefix}.in_proj_weight': (3 * D, D), f'{prefix}.in_proj_bias': (3 * D,),
            f'{prefix}.out_proj.weight': (D, D), f'{prefix}.out_proj.bias': (D,)}


def _ffn_norms(prefix, n_norm):
    s = {f'{prefix}.linear1.weight': (FF, D), f'{prefix}.linear1.bias': (FF,),
         f'{prefix}.linear2.weight': (D, FF), f'{prefix}.linear2.bias': (D,)}
    for i in range(1, n_norm + 1):
        s[f'{prefix}.norm{i}.weight'] = (D,)
        s[f'{prefix}.norm{i}.bias'] = (D,)
    return s


def _enc_layer(prefix):
    return {**_attn(prefix + '.self_attn'), **_ffn_norms(prefix, 2)}


def _dec_layer(prefix):
    return {**_attn(prefix + '.self_attn'), **_attn(prefix + '.multihead_attn'), **_ffn_norms(prefix, 3)}


def _linear(prefix, dout, din):
    return {f'{prefix}.weight': (dout, din), f'{prefix}.bias': (dout,)}


def _mlp(prefix, din, hdims):
    s = {}
    for i, h in enumerate(hdims):
        s.update(_linear(f'{prefix}.affine_layers.{i}', h, din))
        din = h
    return s


def infiller_param_shapes():
    s = {}
    s.update(_linear('context_encoder.in_fc', D, 69))
    s.update(_linear('context_encoder.pos_enc.fc', D, 2 * D))
    for l in range(2):
        s.update(_enc_layer(f'context_encoder.temporal_net.layers.{l}'))
    s.update(_linear('data_decoder.pos_enc.fc', D, D + NZ))
    for l in range(2):
        s.update(_dec_layer(f'data_decoder.temporal_net.layers.{l}'))
    s.update(_mlp('data_decoder.out_mlp', D, [512, 256]))
    s.update(_linear('data_decoder.out_fc', 69, D))
    s.update(_linear('data_decoder.prior_pos_enc.fc', D, 2 * D))
    s.update(_dec_layer('data_decoder.prior_temporal_net.layers.0'))
    s['data_decoder.mu_token'] = (D,)
    s['data_decoder.logvar_token'] = (D,)
    s.update(_linear('data_decoder.p_z_mu_net', NZ, D))
    s.update(_linear('data_decoder.p_z_logvar_net', NZ, D))
    return s


def infiller_posterior_param_shapes():
    """the infiller's posterior encoder q(z | X, C) (DataEncoder, motion_infiller_vae.py:126-249), which only reconstruction runs.
    Kept apart from infiller_param_shapes(): make_state draws the sorted names from one stream, so a new name there would move
    every other stand-in weight."""
    s = {}
    s.update(_linear('data_encoder.in_fc', D, 69))
    s.update(_linear('data_encoder.pos_enc.fc', D, 2 * D))
    for l in range(2):
        s.update(_dec_layer(f'data_encoder.temporal_net.layers.{l}'))
    s['data_encoder.mu_token'] = (D,)
    s['data_encoder.logvar_token'] = (D,)
    s.update(_linear('data_encoder.q_z_mu_net', NZ, D))
    s.update(_linear('data_encoder.q_z_logvar_net', NZ, D))
    return s


def make_infiller_posterior_state(seed=1236):
    """stand-in posterior weights from a seed of their own; merged into make_prior_states()[0] they make a full infiller"""
    return make_state(infiller_posterior_param_shapes(), seed)


def trajpred_param_shapes():
    s = {}
    s.update(_mlp('context_encoder.in_mlp', 69, [512, 256]))
    for l in range(2):
        for d in ['rnn_f', 'rnn_b']:
            p = f'context_encoder.temporal_net.{l}.{d}'
            s.update({f'{p}.weight_ih': (512, 256), f'{p}.weight_hh': (512, 128), f'{p}.bias_ih': (512,), f'{p}.bias_hh': (512,)})
    s.update(_mlp('context_encoder.out_mlp', 256, [512, 256]))
    s.update(_mlp('data_decoder.out_mlp', 256 + NZ, [512, 256]))
    s.update(_linear('data_decoder.out_fc', 11, 256))
    s.update(_mlp('data_decoder.prior_mlp', 256, [512, 256]))
    s.update(_linear('data_decoder.p_z_net', 2 * NZ, 256))
    return s


def make_state(shapes, seed):
    """uniform(-1/sqrt(fan_in), 1/sqrt(fan_in)) matrices, small biases, LayerNorm gains around 1"""
    rng = np.random.default_rng(seed)
    state = {}
    for name in sorted(shapes):
        shp = shapes[name]
        if len(shp) == 2:
            k = 1.0 / np.sqrt(shp[1])
            w = rng.uniform(-k, k, shp)
        elif 'norm' in name and name.endswith('weight'):
            w = 1.0 + rng.normal(0.0, 0.05, shp)
        elif 'token' in name:
            w = rng.normal(0.0, 0.5, shp)
        else:
            w = rng.normal(0.0, 0.05, shp)
        state[name] = w.astype(np.float32)
    return state


def make_prior_states(seed=1234):
    return make_state(infiller_param_shapes(), seed), make_state(trajpred_param_shapes(), seed + 1)
