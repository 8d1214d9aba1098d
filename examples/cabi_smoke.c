/*
 * Plain-C user of the C ABI (no Python, no torch): proves that include/s3prl_b200.h is valid C and that every entry
 * point links. On a GPU-less host it only queries the library; with a device it would go on to
 * s3b_model_create / set_tensor / finalize / s3b_forward_host (see INTEGRATION.md for the full sequence).
 *
 *   gcc -std=c99 -Wall -Werror -Iinclude examples/cabi_smoke.c -Ls3prl_b200/_lib -ls3prl_b200 \
 *       -Wl,-rpath,$PWD/s3prl_b200/_lib -o cabi_smoke && ./cabi_smoke
 */
#include <stdio.h>
#include <string.h>

#include "s3prl_b200.h"

int main(void) {
    /* take the address of every entry point so that a missing export fails at link time */
    const void* entry[] = {
        (const void*)s3b_version,        (const void*)s3b_last_error,      (const void*)s3b_device_count,
        (const void*)s3b_model_create,   (const void*)s3b_model_set_tensor, (const void*)s3b_model_finalize,
        (const void*)s3b_model_destroy,  (const void*)s3b_num_frames,      (const void*)s3b_valid_frames,
        (const void*)s3b_forward,        (const void*)s3b_forward_host,    (const void*)s3b_profile_enable,
        (const void*)s3b_profile_read,   (const void*)s3b_launch_count,    (const void*)s3b_weighted_sum,
        (const void*)s3b_weighted_sum_backward, (const void*)s3b_fbank,    (const void*)s3b_fbank_num_frames,
        (const void*)s3b_trimmed_lengths, (const void*)s3b_melspec,        (const void*)s3b_linear_f32,
        (const void*)s3b_layernorm_f32,  (const void*)s3b_attention_f32,  (const void*)s3b_forward_ex,
        (const void*)s3b_forward_host_ex, (const void*)s3b_wavlm_buckets, (const void*)s3b_peer_create,
        (const void*)s3b_peer_connect,   (const void*)s3b_peer_slot,       (const void*)s3b_peer_push,
        (const void*)s3b_peer_wait,      (const void*)s3b_peer_destroy,    (const void*)s3b_gemm_bench,
        (const void*)s3b_num_outputs,    (const void*)s3b_default_lanes,   (const void*)s3b_attention_ex,
        (const void*)s3b_wavlm_gate_f32, (const void*)s3b_linear_ex,      (const void*)s3b_qkv_f32,
        (const void*)s3b_conv_gemm_f32,  (const void*)s3b_posconv_f32,    (const void*)s3b_frontend_f32,
        (const void*)s3b_conformer_conv_f32, (const void*)s3b_layernorm_rope_f32, (const void*)s3b_qkv_hd_f32,
        (const void*)s3b_fbank_ex,       (const void*)s3b_melspec_ex,     (const void*)s3b_decoar2_features_f32,
        (const void*)s3b_apc_model_create, (const void*)s3b_profile_read_ex, (const void*)s3b_apc_features_f32,
        (const void*)s3b_gru_f32,        (const void*)s3b_gru_max_active_clusters,
        (const void*)s3b_decoar_model_create, (const void*)s3b_lstm_f32, (const void*)s3b_lstm_fits,
        (const void*)s3b_npc_model_create, (const void*)s3b_npc_conv_f32,
        (const void*)s3b_cpc_model_create, (const void*)s3b_cpc_conv_f32, (const void*)s3b_cpc_lstm_f32,
        (const void*)s3b_cpc_lstm_max_active_clusters, (const void*)s3b_ssast_model_create,
        (const void*)s3b_layernorm_eps_f32, (const void*)s3b_ssast_fbank_f32, (const void*)s3b_ssast_embed_f32,
        (const void*)s3b_ssast_fold_f32, (const void*)s3b_layernorm_eps_planes_f32, (const void*)s3b_fbank_cmvn_planes,
        (const void*)s3b_mae_ast_model_create, (const void*)s3b_mae_ast_fbank_f32, (const void*)s3b_mae_ast_embed_f32,
        (const void*)s3b_ssast_patch_planes, (const void*)s3b_mae_ast_fbank_planes,
    };
    s3b_config cfg;
    int64_t lens[2] = {16000, 800};
    int32_t valid[2] = {0, 0};
    memset(&cfg, 0, sizeof(cfg));
    printf("s3prl_b200 C ABI version %d, %d entry points, %d CUDA device(s)\n", s3b_version(),
           (int)(sizeof(entry) / sizeof(entry[0])), s3b_device_count());
    /* integer rules need no device: frames of a 1 s utterance; HuBERT frame-mask rule (hubert_model.py:454-464) for a
     * ragged pair, through a model handle that is never finalized (no GPU needed until s3b_model_finalize) */
    if (s3b_num_frames(NULL, 16000) != 49) return 1;
    cfg.family = 0, cfg.num_layers = 12, cfg.embed_dim = 768, cfg.ffn_dim = 3072, cfg.num_heads = 12;
    cfg.pos_conv_kernel = 128, cfg.pos_conv_groups = 16;
    {
        s3b_model* m = NULL;
        if (s3b_model_create(&cfg, &m) != 0) {
            printf("s3b_model_create: %s\n", s3b_last_error());
            return 2;
        }
        if (s3b_valid_frames(m, lens, 2, 16000, valid) != 0) {
            printf("s3b_valid_frames: %s\n", s3b_last_error());
            return 3;
        }
        printf("valid frames of (16000, 800) samples: %d %d\n", (int)valid[0], (int)valid[1]);
        s3b_model_destroy(m);
        if (valid[0] != 49 || valid[1] != 3) return 4; /* 800 samples cover frames 0..2 (chunks of 326 samples) */
    }
    {
        /* APC: one frame per kaldi fbank frame, 1 + (n - 400) / 160 */
        s3b_apc_config acfg;
        s3b_model* m = NULL;
        memset(&acfg, 0, sizeof(acfg));
        acfg.struct_size = (int32_t)sizeof(acfg), acfg.num_layers = 3, acfg.hidden = 512, acfg.residual = 1;
        if (s3b_apc_model_create(&acfg, &m) != 0) {
            printf("s3b_apc_model_create: %s\n", s3b_last_error());
            return 5;
        }
        if (s3b_valid_frames(m, lens, 2, 16000, valid) != 0 || s3b_num_outputs(m) != 3) {
            printf("APC bookkeeping: %s\n", s3b_last_error());
            return 6;
        }
        printf("APC frames of (16000, 800) samples: %d %d\n", (int)valid[0], (int)valid[1]);
        s3b_model_destroy(m);
        if (valid[0] != 98 || valid[1] != 3) return 7;
    }
    {
        /* DeCoAR: the APC frame rule; decoar outputs the last layer, decoar_layers all four */
        s3b_decoar_config dcfg;
        int32_t all;
        for (all = 0; all < 2; ++all) {
            s3b_model* m = NULL;
            memset(&dcfg, 0, sizeof(dcfg));
            dcfg.struct_size = (int32_t)sizeof(dcfg), dcfg.num_layers = 4, dcfg.hidden = 1024, dcfg.all_layers = all;
            if (s3b_decoar_model_create(&dcfg, &m) != 0) {
                printf("s3b_decoar_model_create: %s\n", s3b_last_error());
                return 8;
            }
            if (s3b_valid_frames(m, lens, 2, 16000, valid) != 0 || s3b_num_outputs(m) != (all ? 4 : 1)) {
                printf("DeCoAR bookkeeping: %s\n", s3b_last_error());
                return 9;
            }
            s3b_model_destroy(m);
            if (valid[0] != 98 || valid[1] != 3) return 10;
        }
    }
    {
        /* NPC: the APC frame rule; every block, every masked conv and feat are outputs (4 blocks: 9) */
        s3b_npc_config ncfg;
        s3b_model* m = NULL;
        memset(&ncfg, 0, sizeof(ncfg));
        ncfg.struct_size = (int32_t)sizeof(ncfg), ncfg.n_blocks = 4, ncfg.hidden = 512;
        ncfg.kernel_size = 15, ncfg.mask_size = 5, ncfg.residual = 1, ncfg.batch_norm = 1, ncfg.act = 0;
        if (s3b_npc_model_create(&ncfg, &m) != 0) {
            printf("s3b_npc_model_create: %s\n", s3b_last_error());
            return 11;
        }
        if (s3b_valid_frames(m, lens, 2, 16000, valid) != 0 || s3b_num_outputs(m) != 9) {
            printf("NPC bookkeeping: %s\n", s3b_last_error());
            return 12;
        }
        s3b_model_destroy(m);
        if (valid[0] != 98 || valid[1] != 3) return 13;
    }
    {
        /* modified CPC: the padded conv chain (16000 -> 100, 800 -> 5); the encoder and the last LSTM layer */
        s3b_cpc_config ccfg;
        s3b_model* m = NULL;
        memset(&ccfg, 0, sizeof(ccfg));
        ccfg.struct_size = (int32_t)sizeof(ccfg), ccfg.hidden = 256, ccfg.num_layers = 1;
        if (s3b_cpc_model_create(&ccfg, &m) != 0) {
            printf("s3b_cpc_model_create: %s\n", s3b_last_error());
            return 14;
        }
        if (s3b_valid_frames(m, lens, 2, 16000, valid) != 0 || s3b_num_outputs(m) != 2 ||
            s3b_num_frames(m, 16000) != 100 || s3b_num_frames(m, 158) != -1) {
            printf("CPC bookkeeping: %s\n", s3b_last_error());
            return 15;
        }
        s3b_model_destroy(m);
        if (valid[0] != 100 || valid[1] != 5) return 16;
    }
    {
        /* LightHuBERT small: 384 channels, 16 pos_conv groups of 24, hidden state 0 = post_extract_proj's output; the
         * HuBERT frame rule */
        s3b_model* m = NULL;
        memset(&cfg, 0, sizeof(cfg));
        cfg.family = 0, cfg.extractor_layer_norm = 1, cfg.normalize_wav = 1, cfg.num_layers = 12, cfg.embed_dim = 384;
        cfg.ffn_dim = 1536, cfg.num_heads = 6, cfg.pos_conv_kernel = 128, cfg.pos_conv_groups = 16, cfg.proj_hidden0 = 1;
        if (s3b_model_create(&cfg, &m) != 0) {
            printf("s3b_model_create (LightHuBERT): %s\n", s3b_last_error());
            return 17;
        }
        if (s3b_valid_frames(m, lens, 2, 16000, valid) != 0 || s3b_num_outputs(m) != 13) {
            printf("LightHuBERT bookkeeping: %s\n", s3b_last_error());
            return 18;
        }
        s3b_model_destroy(m);
        if (valid[0] != 49 || valid[1] != 3) return 19;
    }
    {
        /* SSAST frame model, 1 s windows: 99 frames per window, trimmed to ceil(max_len / 160); 12 block outputs */
        s3b_ssast_config scfg;
        s3b_model* m = NULL;
        memset(&scfg, 0, sizeof(scfg));
        scfg.struct_size = (int32_t)sizeof(scfg), scfg.patch = 0, scfg.window_samples = 16000;
        scfg.embed_dim = 768, scfg.num_heads = 12, scfg.num_layers = 12;
        if (s3b_ssast_model_create(&scfg, &m) != 0) {
            printf("s3b_ssast_model_create: %s\n", s3b_last_error());
            return 20;
        }
        if (s3b_valid_frames(m, lens, 2, 16000, valid) != 0 || s3b_num_outputs(m) != 12 ||
            s3b_num_frames(m, 16000) != 99 || s3b_num_frames(m, 16001) != 101) {
            printf("SSAST bookkeeping: %s\n", s3b_last_error());
            return 21;
        }
        s3b_model_destroy(m);
        if (valid[0] != 99 || valid[1] != 5) return 22;
    }
    {
        /* MAE-AST frame model: 99 fbank frames -> 49 patches of 2; 800 samples = 3 frames -> 2 valid patches */
        s3b_mae_ast_config mcfg;
        s3b_model* m = NULL;
        memset(&mcfg, 0, sizeof(mcfg));
        mcfg.struct_size = (int32_t)sizeof(mcfg), mcfg.patch = 0, mcfg.embed_dim = 768, mcfg.num_heads = 12;
        mcfg.ffn_dim = 3072, mcfg.num_layers = 12, mcfg.sine_pos = 1, mcfg.max_tokens = 48000;
        if (s3b_mae_ast_model_create(&mcfg, &m) != 0) {
            printf("s3b_mae_ast_model_create: %s\n", s3b_last_error());
            return 23;
        }
        if (s3b_valid_frames(m, lens, 2, 16000, valid) != 0 || s3b_num_outputs(m) != 12 || s3b_num_frames(m, 16000) != 49) {
            printf("MAE-AST bookkeeping: %s\n", s3b_last_error());
            return 24;
        }
        s3b_model_destroy(m);
        if (valid[0] != 49 || valid[1] != 2) return 25;
    }
    return 0;
}
