// B200Native.cs -- the B200 backend of the CryptoNets plugin API: every member of IFactory (HE Wrapper/IFactory.cs:20-130), IVector
// (HE Wrapper/IVector.cs:20-136), IMatrix (HE Wrapper/IMatrix.cs:18-122) and IComputationEnvironment over P/Invoke into libcnhe.so
// (include/cnhe.h).  A maintainer drops this file next to HE Wrapper/IFactory.cs and changes the factory constructor line of an app
// (CryptoNets/CryptoNets.cs:17, LowLatencyCryptoNets/LoLaCryptonets.cs:285, ...) from `new EncryptedSealBfvFactory(...)` to
// `new B200BfvFactory(...)`; layers and apps are otherwise untouched.
//
// NOT COMPILED IN THIS REPOSITORY: the build image has no .NET toolchain (SURVEY.md section 0).  tools/check_csharp_bindings.py checks
// every [DllImport] below against include/cnhe.h (name, arity, parameter types) and that every interface member of the three reference
// interfaces is implemented here; the Python mirror with the same member names (cryptonets_b200/he.py) is what the tests drive.
using MathNet.Numerics.LinearAlgebra;
using System;
using System.Collections.Generic;
using System.IO;
using System.Linq;
using System.Numerics;
using System.Runtime.InteropServices;
using System.Text;

namespace HEWrapper
{
    internal static class Cnhe
    {
        const string Lib = "cnhe"; // libcnhe.so / cnhe.dll
        public const ulong AllSlots = 0x7FFFFFFF; // CNHE_ALL_SLOTS
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern IntPtr cnhe_last_error();
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern IntPtr cnhe_version();
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_create(ulong[] plain_primes, int P, uint N, int dbc_relin, int dbc_galois, int small_modulus_count, int device, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_create_custom(ulong[] plain_primes, int P, uint N, ulong[] coeff_moduli, int k, int dbc_relin, int dbc_galois, int device, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_destroy(IntPtr a0);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_info(IntPtr a0, out uint N, out int k, out int P, out int relin_digits, out int galois_digits, out int galois_elts);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_coeff_moduli(IntPtr a0, ulong[] out_k);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_plain_moduli(IntPtr a0, ulong[] out_P);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_bsk_moduli(IntPtr a0, ulong[] @out, out int count);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_product_sum_terms(IntPtr a0, out int terms);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_galois_elts(IntPtr a0, ulong[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_set_option(IntPtr a0, string name, long value);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_sync(IntPtr a0);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_stream(IntPtr a0, int channel, out ulong stream);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_join_streams(IntPtr a0);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_fork_streams(IntPtr a0);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_keys_generate_secure(IntPtr a0);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_keys_generate(IntPtr a0, ulong seed);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_keys_export(IntPtr a0, int channel, int what, ulong arg, IntPtr dst, UIntPtr cap_words);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_keys_import(IntPtr a0, int channel, int what, ulong arg, IntPtr src, UIntPtr words);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_keys_set_seed(IntPtr a0, int channel, ulong seed);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_op_counts(IntPtr a0, ulong[] @out, int cap, int reset);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern IntPtr cnhe_op_name(int kind);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_trace_read(IntPtr a0, int[] @out, UIntPtr cap_records, out UIntPtr n_records, int clear);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_keys_save(IntPtr a0, int with_private_keys, byte[] dst, UIntPtr cap, out UIntPtr needed);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_load(byte[] archive, UIntPtr len, int device, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_keys_save_compact(IntPtr a0, int sets, ulong[] galois_elts, int n_galois, byte[] dst, UIntPtr cap, out UIntPtr needed);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_load_compact(byte[] blob, UIntPtr len, int device, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_add_client_compact(IntPtr a0, byte[] blob, UIntPtr len, out int slot);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_remove_client(IntPtr a0, int slot);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_set_key_slot(IntPtr a0, int slot);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_key_slot(IntPtr a0, out int slot);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_context_derive_level(IntPtr a0, int k, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_mod_switch(IntPtr from, IntPtr[] @in, int n, IntPtr to, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_sanitize(IntPtr ctx, IntPtr[] @in, int n, int flood_bits, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_write(IntPtr a0, IntPtr a1, byte[] dst, UIntPtr cap, out UIntPtr needed);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_read(IntPtr a0, byte[] text, UIntPtr len, out IntPtr @out, out UIntPtr consumed);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_encrypt(IntPtr a0, double[] v, ulong dim, double scale, int format, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_plain(IntPtr a0, double[] v, ulong dim, double scale, int format, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_encrypt(IntPtr a0, double[] v, int n, ulong dim, double scale, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_decrypt(IntPtr a0, IntPtr a1, double[] @out, ulong cap);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_decrypt(IntPtr a0, IntPtr[] vecs, int n, double[] @out, ulong dim);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_copy(IntPtr a0, IntPtr a1, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_destroy(IntPtr a0);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_destroy(IntPtr[] vecs, int n);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_meta(IntPtr a0, out ulong dim, out double scale, out int format, out int is_encrypted, out int blocks, out ulong block_size);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_register_scale(IntPtr a0, double scale);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_register_dim(IntPtr a0, ulong dim);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_export_raw(IntPtr a0, IntPtr a1, int channel, int block, IntPtr dst, UIntPtr cap_words);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_import_raw(IntPtr a0, IntPtr src, int blocks, ulong dim, double scale, int format, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_import_raw(IntPtr a0, IntPtr src, int n, int blocks, ulong dim, double scale, int format, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_export_raw(IntPtr a0, IntPtr[] vecs, int n, IntPtr dst, UIntPtr cap_words);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_export_raw_async(IntPtr a0, IntPtr[] vecs, int n, IntPtr dst, UIntPtr cap_words, out int ticket);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_export_wait(IntPtr a0, int ticket);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_encrypt_compact(IntPtr a0, double[] v, int n, ulong dim, double scale, byte[] dst, UIntPtr cap, out UIntPtr needed);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_import_compact(IntPtr a0, byte[] src, UIntPtr len, IntPtr[] @out, int cap, out int n);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_encrypt_device(IntPtr a0, ulong d_values, int n, ulong dim, double scale, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_encrypt_compact_device(IntPtr a0, ulong d_values, int n, ulong dim, double scale, byte[] dst, UIntPtr cap, out UIntPtr needed);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_decrypt_device(IntPtr a0, IntPtr[] vecs, int n, ulong d_out, ulong dim);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_device_ptr(IntPtr a0, int channel, out ulong dptr, out UIntPtr words);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_noise_budget(IntPtr a0, IntPtr a1, int channel, int block, out int bits);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_add(IntPtr a0, IntPtr a, IntPtr b, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_sub(IntPtr a0, IntPtr a, IntPtr b, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_pointwise_multiply(IntPtr a0, IntPtr a, IntPtr b, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_sum_all_slots(IntPtr a0, IntPtr a, ulong length, int force_column, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_dot_product(IntPtr a0, IntPtr a, IntPtr b, ulong length, int force_column, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_rotate(IntPtr a0, IntPtr a, int amount, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_duplicate(IntPtr a0, IntPtr a, ulong count, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_permute(IntPtr a0, IntPtr a, IntPtr[] selections, int[] shifts, int n, ulong output_dim, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_interleave(IntPtr a0, IntPtr[] vecs, int n, int shift, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_stack(IntPtr a0, IntPtr[] vecs, int n, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_generate_sparse_of_array(IntPtr a0, IntPtr[] vecs, int n, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_rotate(IntPtr a0, IntPtr[] vecs, int n, int amount, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_stack_batch(IntPtr a0, IntPtr[] vecs, int n, int B, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_mat_mul_colmajor_sparse(IntPtr a0, IntPtr[] cols, int K, IntPtr sparse, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_mat_mul_colmajor_sparse_deferred(IntPtr a0, IntPtr[] cols, int K, IntPtr sparse, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_mat_mul_rowmajor(IntPtr a0, IntPtr[] rows, int n_rows, IntPtr v, int force_dense, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_mat_mul_rowmajor_batch(IntPtr a0, IntPtr[] rows, int n_rows, IntPtr[] vs, int B, int force_dense, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_mat_dot_rows_batch(IntPtr a0, IntPtr[] rows, int n_rows, IntPtr[] vs, int B, ulong length, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_duplicate_batch(IntPtr a0, IntPtr[] vecs, int B, ulong count, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_permute_batch(IntPtr a0, IntPtr[] vecs, int B, IntPtr[] selections, int[] shifts, int n_perm, int n_sel, ulong output_dim, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_interleave_batch(IntPtr a0, IntPtr[] vecs, int n, int B, int shift, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_multiply_plain(IntPtr a0, IntPtr[] vecs, int n, IntPtr plain, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_mat_mul_rowmajor_shard(IntPtr a0, IntPtr[] rows, int n_rows, IntPtr v, int force_dense, int first_row, int total_rows, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_diag_prepare(IntPtr a0, IntPtr[] rows, int n_rows, int baby_steps, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_diag_info(IntPtr a0, out int n_rows, out ulong dim, out int n1, out int n2, out int n_diags, out ulong device_bytes);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_diag_export(IntPtr a0, IntPtr diag, int channel, int index, ulong[] dst, UIntPtr cap_words, int[] bgh);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_diag_destroy(IntPtr a0);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_diag_prepare_ntt(IntPtr a0, IntPtr[] rows, int n_rows, int baby_steps, ulong max_ntt_bytes, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_diag_ntt_info(IntPtr a0, out int resident_giant_steps, out int resident_diags, out ulong ntt_bytes);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_diag_export_ntt(IntPtr a0, IntPtr diag, int channel, int index, ulong[] dst, UIntPtr cap_words);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_mat_mul_diagonal(IntPtr a0, IntPtr diag, IntPtr[] vs, int B, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_diag_prepare_folded(IntPtr a0, IntPtr[] rows, int n_rows, int fold_width, int baby_steps, ulong max_ntt_bytes, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_diag_fold_width(IntPtr a0, out int width);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_layer_conv_dense(IntPtr a0, IntPtr[] @in, int n_in, int[] gather, IntPtr[] weights, IntPtr[] bias, int M, int K, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_layer_square(IntPtr a0, IntPtr[] @in, int n, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_layer_poly2(IntPtr a0, IntPtr[] @in, int n, IntPtr a, IntPtr b, IntPtr c, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_layer_poly(IntPtr a0, IntPtr[] @in, int n, IntPtr[] coeffs, int degree, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_layer_activation_conv_dense(IntPtr a0, IntPtr[] @in, int n_in, IntPtr a, IntPtr b, IntPtr c, int[] gather, IntPtr[] weights, IntPtr[] bias, int M, int K, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_dev_alloc(IntPtr a0, UIntPtr words, out ulong dptr);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_dev_free(IntPtr a0, ulong dptr);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_dev_upload(IntPtr a0, ulong dptr, IntPtr src, UIntPtr words);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_dev_download(IntPtr a0, IntPtr dst, ulong dptr, UIntPtr words);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_raw_ntt(IntPtr a0, ulong src, ulong dst, int n_polys, int mod_base, int mod_count, int inverse);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_raw_multiply(IntPtr a0, int channel, ulong a, ulong b, int n, ulong out3);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_raw_relinearize(IntPtr a0, int channel, ulong in3, int n, ulong out2);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_raw_multiply_relin(IntPtr a0, int channel, ulong a, ulong b, int n, ulong out2);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_raw_apply_galois(IntPtr a0, int channel, ulong @in, int n, ulong galois_elt, ulong @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_raw_rotate_rows(IntPtr a0, int channel, ulong @in, int n, int steps, ulong @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_raw_behz_lift(IntPtr a0, ulong in_cts, int n, ulong out_together);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_raw_behz_floor(IntPtr a0, int channel, ulong d_together, int n, ulong out3);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_dev_copy(IntPtr a0, ulong dst, ulong src, UIntPtr words);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_raw_import_products(IntPtr a0, ulong[] words, int n, ulong dim, double scale, int slot, IntPtr[] @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_prof_enable(IntPtr a0, int on);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_prof_collect(IntPtr a0, int family, out double total_ms, out ulong launches, out double algorithmic_bytes);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_raw_event_timing(IntPtr a0, int start);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_raw_elapsed_ms(IntPtr a0, out float ms);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern ulong cnhe_kernel_launch_count(IntPtr a0);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_capture_begin(IntPtr a0);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_capture_begin_levels(IntPtr ctx, IntPtr[] levels, int n);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_capture_end(IntPtr a0, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_capture_abort(IntPtr a0);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_graph_launch(IntPtr a0);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_graph_slots(IntPtr a0, int[] slots, int cap, out int n);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_graph_bind(IntPtr a0, int[] slots, int n);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_graph_info(IntPtr a0, out ulong kernel_nodes, out ulong device_bytes);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_graph_destroy(IntPtr a0);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vecs_assign(IntPtr a0, IntPtr[] dst, IntPtr[] src, int n);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_from_residues(IntPtr a0, ulong[] residues, ulong dim, double scale, int format, int encrypt, out IntPtr @out);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int cnhe_vec_decrypt_residues(IntPtr a0, IntPtr a1, ulong[] @out, ulong cap_words);

        /// the reference throws System.Exception("...") on every misuse (e.g. AtomicSealBfvVector.cs:987-991); keep that contract
        public static void Check(int rc)
        {
            if (rc != 0) throw new Exception(Marshal.PtrToStringAnsi(cnhe_last_error()));
        }
        public static IntPtr[] Handles(IEnumerable<IVector> vs) => vs.Select(v => v == null ? IntPtr.Zero : ((B200BfvVector)v).Handle).ToArray();
    }

    /// IComputationEnvironment (IComputationEnvironment.cs:12-24).  All environments of a factory share the context's CUDA streams; the
    /// object exists so that reference call sites (Utils.ProcessInEnv, layer code) keep their shape.
    public class B200BfvEnvironment : IComputationEnvironment
    {
        public IFactory ParentFactory { get; internal set; }
        public ulong[] Primes => ((B200BfvFactory)ParentFactory).Primes;
    }

    /// IVector over a device-resident cnhe_vec (== EncryptedSealBfvVector, EncryptedSealBfvVector.cs:150-573)
    public class B200BfvVector : IVector
    {
        internal IntPtr Handle;
        internal readonly B200BfvFactory Factory;
        internal B200BfvVector(B200BfvFactory f, IntPtr h) { Factory = f; Handle = h; }
        IntPtr Ctx => Factory.Ctx;
        B200BfvVector Wrap(IntPtr h) => new B200BfvVector(Factory, h);
        static IntPtr H(IVector v)
        {
            if (!(v is B200BfvVector b)) throw new Exception("expecting B200BfvVector");
            return b.Handle;
        }
        void Meta(out ulong dim, out double scale, out int format, out int enc, out int blocks, out ulong blockSize) =>
            Cnhe.Check(Cnhe.cnhe_vec_meta(Handle, out dim, out scale, out format, out enc, out blocks, out blockSize));

        public object Data => Handle;
        public ulong Dim { get { Meta(out var d, out _, out _, out _, out _, out _); return d; } }
        public double Scale { get { Meta(out _, out var s, out _, out _, out _, out _); return s; } }
        public EVectorFormat Format { get { Meta(out _, out _, out var f, out _, out _, out _); return (EVectorFormat)f; } }
        public bool IsEncrypted { get { Meta(out _, out _, out _, out var e, out _, out _); return e != 0; } }
        public ulong BlockSize { get { Meta(out _, out _, out _, out _, out _, out var b); return b; } }
        public bool IsSigned { get; set; } = true;
        public void RegisterScale(double scale) => Cnhe.Check(Cnhe.cnhe_vec_register_scale(Handle, scale));
        public void RegisterDim(ulong dim) => Cnhe.Check(Cnhe.cnhe_vec_register_dim(Handle, dim));

        public Vector<double> Decrypt(IComputationEnvironment env)
        {
            var dst = new double[Dim];
            Cnhe.Check(Cnhe.cnhe_vec_decrypt(Ctx, Handle, dst, (ulong)dst.Length));
            return Vector<double>.Build.DenseOfArray(dst);
        }
        /// EncryptedSealBfvVector.cs:343-348 + JoinSplitNumbers :397-411 (big-integer CRT join of the per-prime residues)
        public IEnumerable<BigInteger> DecryptFullPrecision(IComputationEnvironment env)
        {
            ulong dim = Dim;
            var primes = Factory.Primes;
            var res = new ulong[dim * (ulong)primes.Length];
            Cnhe.Check(Cnhe.cnhe_vec_decrypt_residues(Ctx, Handle, res, (ulong)res.Length));
            var outv = new BigInteger[dim];
            for (ulong j = 0; j < dim; j++)
            {
                BigInteger x = 0;
                for (int i = 0; i < primes.Length; i++) x += Factory.PreComputedCoefficients[i] * res[(ulong)i * dim + j];
                x %= Factory.BigFactor;
                if (IsSigned && x * 2 > Factory.BigFactor) x -= Factory.BigFactor;
                outv[j] = x;
            }
            return outv;
        }
        public void Write(StreamWriter str)
        {
            Cnhe.Check(Cnhe.cnhe_vec_write(Ctx, Handle, null, UIntPtr.Zero, out var needed));
            var buf = new byte[(int)needed];
            Cnhe.Check(Cnhe.cnhe_vec_write(Ctx, Handle, buf, needed, out needed));
            str.Write(Encoding.ASCII.GetString(buf));
            str.Flush();
        }
        public IVector Subtract(IVector v, IComputationEnvironment env) { Cnhe.Check(Cnhe.cnhe_vec_sub(Ctx, Handle, H(v), out var r)); return Wrap(r); }
        public IVector Add(IVector v, IComputationEnvironment env) { Cnhe.Check(Cnhe.cnhe_vec_add(Ctx, Handle, H(v), out var r)); return Wrap(r); }
        public IVector PointwiseMultiply(IVector v, IComputationEnvironment env) { Cnhe.Check(Cnhe.cnhe_vec_pointwise_multiply(Ctx, Handle, H(v), out var r)); return Wrap(r); }
        public IVector DotProduct(IVector v, IComputationEnvironment env) { Cnhe.Check(Cnhe.cnhe_vec_dot_product(Ctx, Handle, H(v), Cnhe.AllSlots, -1, out var r)); return Wrap(r); }
        public IVector DotProduct(IVector v, ulong length, IComputationEnvironment env) { Cnhe.Check(Cnhe.cnhe_vec_dot_product(Ctx, Handle, H(v), length, -1, out var r)); return Wrap(r); }
        /// EncryptedSealBfvVector.DotProduct(v, env, ForceOutputInColumn) used by EncryptedSealBfvMatrix.Mul (:92-116)
        internal IVector DotProduct(IVector v, IComputationEnvironment env, int forceOutputInColumn) { Cnhe.Check(Cnhe.cnhe_vec_dot_product(Ctx, Handle, H(v), Cnhe.AllSlots, forceOutputInColumn, out var r)); return Wrap(r); }
        public IVector SumAllSlots(IComputationEnvironment env) { Cnhe.Check(Cnhe.cnhe_vec_sum_all_slots(Ctx, Handle, Cnhe.AllSlots, -1, out var r)); return Wrap(r); }
        public IVector Duplicate(ulong count, IComputationEnvironment env) { Cnhe.Check(Cnhe.cnhe_vec_duplicate(Ctx, Handle, count, out var r)); return Wrap(r); }
        public IVector Rotate(int amount, IComputationEnvironment env) { Cnhe.Check(Cnhe.cnhe_vec_rotate(Ctx, Handle, amount, out var r)); return Wrap(r); }
        public IVector Permute(IVector[] selections, int[] shifts, ulong outputDim, IComputationEnvironment env)
        {
            Cnhe.Check(Cnhe.cnhe_vec_permute(Ctx, Handle, Cnhe.Handles(selections), shifts, shifts.Length, outputDim, out var r));
            return Wrap(r);
        }
        public void Dispose()
        {
            if (Handle != IntPtr.Zero) { Cnhe.cnhe_vec_destroy(Handle); Handle = IntPtr.Zero; }
            GC.SuppressFinalize(this);
        }
        ~B200BfvVector() { if (Handle != IntPtr.Zero) Cnhe.cnhe_vec_destroy(Handle); }
    }

    /// IMatrix as an array of vectors (EncryptedSealBfvMatrix.cs:14-231)
    public class B200BfvMatrix : IMatrix
    {
        internal B200BfvVector[] Vectors;
        readonly B200BfvFactory Factory;
        public EMatrixFormat Format { get; private set; }
        public bool DataDisposedExternaly { get; set; } = false;

        internal B200BfvMatrix(B200BfvFactory f, IVector[] vectors, EMatrixFormat format, bool copyVectors)
        {
            if (vectors.Any(v => v.Dim != vectors[0].Dim)) throw new Exception("all columns of a matrix should have the same size");
            Factory = f;
            Format = format;
            Vectors = vectors.Select(v => copyVectors ? (B200BfvVector)f.CopyVector(v) : (B200BfvVector)v).ToArray();
            DataDisposedExternaly = !copyVectors; // EncryptedSealBfvMatrix.cs:37-47
        }
        IntPtr Ctx => Factory.Ctx;
        public object Data => Vectors;
        public ulong RowCount => Format == EMatrixFormat.RowMajor ? (ulong)Vectors.Length : Vectors[0].Dim;
        public ulong ColumnCount => Format == EMatrixFormat.ColumnMajor ? (ulong)Vectors.Length : Vectors[0].Dim;
        public double Scale => Vectors[0].Scale;
        public ulong BlockSize => Vectors[0].BlockSize;
        public bool IsEncrypted => Vectors.All(v => v.IsEncrypted);
        public void RegisterScale(double scale) { foreach (var v in Vectors) v.RegisterScale(scale); }

        public Matrix<double> Decrypt(IComputationEnvironment env)
        {   // EncryptedSealBfvMatrix.cs:60-68
            var vecs = Vectors.Select(v => v.Decrypt(env)).ToArray();
            return Format == EMatrixFormat.ColumnMajor ? Matrix<double>.Build.DenseOfColumnVectors(vecs) : Matrix<double>.Build.DenseOfRowVectors(vecs);
        }
        public void Write(StreamWriter str)
        {   // EncryptedSealBfvMatrix.cs:199-208
            str.WriteLine("<Start LargeEncryptedMatrix>");
            str.WriteLine(Enum.GetName(Format.GetType(), Format));
            str.WriteLine(Vectors.Length);
            foreach (var v in Vectors) v.Write(str);
            str.WriteLine("<End LargeEncryptedMatrix>");
            str.Flush();
        }
        // B200-specific: an encrypted column-major matrix times an encrypted sparse vector with one relinearisation per output block
        // (cnhe_mat_mul_colmajor_sparse_deferred; decrypts to Mul's values)
        public IVector MulDeferred(IVector v)
        {
            if (!(v is B200BfvVector bv)) throw new Exception("expecting B200BfvVector");
            if (Format != EMatrixFormat.ColumnMajor || !IsEncrypted || !bv.IsEncrypted)
                throw new Exception("MulDeferred serves an encrypted column-major matrix times an encrypted sparse vector; use Mul");
            Cnhe.Check(Cnhe.cnhe_mat_mul_colmajor_sparse_deferred(Ctx, Cnhe.Handles(Vectors), Vectors.Length, bv.Handle, out IntPtr r));
            return new B200BfvVector(Factory, r);
        }
        public IVector Mul(IVector v, IComputationEnvironment env, bool ForceDenseFormat = false)
        {   // EncryptedSealBfvMatrix.cs:70-121
            if (!(v is B200BfvVector bv)) throw new Exception("expecting B200BfvVector");
            IntPtr r;
            if (Format == EMatrixFormat.ColumnMajor)
            {
                if (ForceDenseFormat) throw new Exception("Forcing dense format is available only in RowMajor mode");
                Cnhe.Check(Cnhe.cnhe_mat_mul_colmajor_sparse(Ctx, Cnhe.Handles(Vectors), Vectors.Length, bv.Handle, out r));
                return new B200BfvVector(Factory, r);
            }
            if (bv.IsEncrypted && !IsEncrypted)
            {   // all rows through each stage together (same ciphertexts as the per-row loop)
                Cnhe.Check(Cnhe.cnhe_mat_mul_rowmajor(Ctx, Cnhe.Handles(Vectors), Vectors.Length, bv.Handle, ForceDenseFormat ? 1 : 0, out r));
                return new B200BfvVector(Factory, r);
            }
            if (!ForceDenseFormat)
            {
                var tmp = Vectors.Select(row => row.DotProduct(v, env)).ToArray();
                Cnhe.Check(Cnhe.cnhe_vecs_generate_sparse_of_array(Ctx, Cnhe.Handles(tmp), tmp.Length, out r));
                foreach (var t in tmp) t.Dispose();
                return new B200BfvVector(Factory, r);
            }
            IVector total = null;
            for (int i = 0; i < Vectors.Length; i++)
            {
                var t = Vectors[i].DotProduct(v, env, i);
                if (total == null) total = t;
                else { var s = total.Add(t, env); total.Dispose(); t.Dispose(); total = s; }
            }
            ((B200BfvVector)total).RegisterDim((ulong)Vectors.Length);
            return total;
        }
        IMatrix Zip(IMatrix m, Func<IVector, IVector, IVector> f)
        {
            if (!(m is B200BfvMatrix o)) throw new Exception("expecting B200BfvMatrix");
            if (o.Format != Format) throw new Exception("matrices should have the same format");
            if (o.Vectors.Length != Vectors.Length) throw new Exception("dimensions do not match");
            return new B200BfvMatrix(Factory, Vectors.Zip(o.Vectors, f).ToArray(), Format, false) { DataDisposedExternaly = false };
        }
        public IMatrix Add(IMatrix m, IComputationEnvironment env) => Zip(m, (a, b) => a.Add(b, env));                               // :123-137
        public IMatrix ElementWiseMultiply(IMatrix m, IComputationEnvironment env) => Zip(m, (a, b) => a.PointwiseMultiply(b, env)); // :140-154
        /// a x^2 + b x + c of every column in one wave (cnhe_layer_poly2): a, b, c plain sparse vectors of dimension 1 at scales W, W s, W s^2
        /// (b, c may be null); the result has scale W s^2
        public IMatrix PolyActivation(IVector a, IVector b, IVector c)
        {
            var outs = new IntPtr[Vectors.Length];
            Cnhe.Check(Cnhe.cnhe_layer_poly2(Ctx, Cnhe.Handles(Vectors), Vectors.Length, ((B200BfvVector)a).Handle,
                                             b == null ? IntPtr.Zero : ((B200BfvVector)b).Handle, c == null ? IntPtr.Zero : ((B200BfvVector)c).Handle, outs));
            return new B200BfvMatrix(Factory, outs.Select(h => (IVector)new B200BfvVector(Factory, h)).ToArray(), Format, false) { DataDisposedExternaly = false };
        }
        /// the cubic or quartic of every column in two levels of squares (cnhe_layer_poly): 4 or 5 plain sparse vectors of dimension 1,
        /// highest degree first (null for 0, the first required), coefficient j at scale W s^(d - j); the result has scale W s^d
        public IMatrix PolyActivation(IVector[] coefficients)
        {
            var outs = new IntPtr[Vectors.Length];
            var coeffs = coefficients.Reverse().Select(v => v == null ? IntPtr.Zero : ((B200BfvVector)v).Handle).ToArray();
            Cnhe.Check(Cnhe.cnhe_layer_poly(Ctx, Cnhe.Handles(Vectors), Vectors.Length, coeffs, coeffs.Length - 1, outs));
            return new B200BfvMatrix(Factory, outs.Select(h => (IVector)new B200BfvVector(Factory, h)).ToArray(), Format, false) { DataDisposedExternaly = false };
        }
        /// the square (a, b, c null) or a x^2 + b x + c of every column followed by the scalar-MAC layer of ConvDenseLayer, relinearising only
        /// the M outputs (cnhe_layer_activation_conv_dense); the outputs have scale scale(a) s^2 scale(w), which the bias must share
        public IVector[] ActivationConvDense(IVector a, IVector b, IVector c, int[] gather, IVector[] weights, IVector[] bias, int M, int K)
        {
            IntPtr H(IVector v) => v == null ? IntPtr.Zero : ((B200BfvVector)v).Handle;
            var outs = new IntPtr[M];
            Cnhe.Check(Cnhe.cnhe_layer_activation_conv_dense(Ctx, Cnhe.Handles(Vectors), Vectors.Length, H(a), H(b), H(c), gather, Cnhe.Handles(weights),
                                                             bias == null ? null : Cnhe.Handles(bias), M, K, outs));
            return outs.Select(h => (IVector)new B200BfvVector(Factory, h)).ToArray();
        }
        public IVector GetColumn(int columnNumber)
        {
            if (Format != EMatrixFormat.ColumnMajor) throw new Exception("GetColumn is available only for ColumnMajor matrices");
            return Vectors[columnNumber];
        }
        public IVector GetRow(int rowNumber)
        {
            if (Format != EMatrixFormat.RowMajor) throw new Exception("GetRow is available only for RowMajor matrices");
            return Vectors[rowNumber];
        }
        public void SetColumn(int columnNumber, IVector vector)
        {   // EncryptedSealBfvMatrix.cs:166-177
            if (Format != EMatrixFormat.ColumnMajor) throw new Exception("Format mismatch");
            if (vector.Dim != Vectors[columnNumber].Dim) throw new Exception("Dimension of vector does not match the dimension of the vector it is replacing");
            if (vector.Scale != Vectors[columnNumber].Scale) throw new Exception("Scale of vector does not match the scale of the vector it is replacing");
            if (vector.IsEncrypted != Vectors[columnNumber].IsEncrypted) throw new Exception("can't exchange encrypted and not encrypted vectors");
            if (!(vector is B200BfvVector v)) throw new Exception("expecting B200BfvVector");
            Vectors[columnNumber] = v;
        }
        public IVector ConvertToColumnVector(IComputationEnvironment env)
        {   // EncryptedSealBfvMatrix.cs:215-220 -> AtomicSealBfvEncryptedVector.Stack
            if (Format != EMatrixFormat.ColumnMajor) throw new Exception("Expecting ColumnMajor matrix");
            Cnhe.Check(Cnhe.cnhe_vecs_stack(Ctx, Cnhe.Handles(Vectors), Vectors.Length, out var r));
            return new B200BfvVector(Factory, r);
        }
        public IVector Interleave(int shift, IComputationEnvironment env)
        {   // EncryptedSealBfvMatrix.cs:221-226
            if (Format != EMatrixFormat.ColumnMajor) throw new Exception("Expecting ColumnMajor matrix");
            Cnhe.Check(Cnhe.cnhe_vecs_interleave(Ctx, Cnhe.Handles(Vectors), Vectors.Length, shift, out var r));
            return new B200BfvVector(Factory, r);
        }
        public void Dispose()
        {
            if (Vectors != null && !DataDisposedExternaly)
            {
                var hs = Vectors.Where(v => v != null && v.Handle != IntPtr.Zero).ToArray();
                if (hs.Length > 0) Cnhe.cnhe_vecs_destroy(hs.Select(v => v.Handle).ToArray(), hs.Length); // one call for the whole matrix
                foreach (var v in hs) { v.Handle = IntPtr.Zero; GC.SuppressFinalize(v); }
            }
            Vectors = null;
        }
    }

    /// IFactory (IFactory.cs:20-130); constructor arguments of EncryptedSealBfvFactory (IFactory.cs:247-271)
    public class B200BfvFactory : IFactory, IDisposable
    {
        internal IntPtr Ctx;
        public ulong[] Primes { get; private set; }
        internal BigInteger BigFactor;
        internal BigInteger[] PreComputedCoefficients; // EncryptedSealBfvEnvironment.PreCompute, EncryptedSealBfvVector.cs:79-90
        readonly B200BfvEnvironment env;

        /// keys come from the OS CSPRNG (cnhe_keys_generate_secure), as SEAL's KeyGenerator gives the reference
        public B200BfvFactory(ulong[] primes = null, ulong n = 4096, int DecompositionBitCount = 10, int GaloisDecompositionBitCount = 20,
                              int SmallModulusCount = -1, int device = 0)
        {
            if (primes == null) { primes = new ulong[] { 40961, 65537, 114689, 147457, 188417 }; n = 4096; } // IFactory.cs:247-253
            Cnhe.Check(Cnhe.cnhe_context_create(primes, primes.Length, (uint)n, DecompositionBitCount, GaloisDecompositionBitCount, SmallModulusCount,
                                                device, out Ctx));
            Cnhe.Check(Cnhe.cnhe_keys_generate_secure(Ctx));
            env = new B200BfvEnvironment { ParentFactory = this };
            SetPrimes(primes);
        }
        /// EncryptedSealBfvFactory(string fileName) (IFactory.cs:262-271): parameters and keys from a key archive written by Save
        public B200BfvFactory(string fileName, int device = 0) : this(File.ReadAllBytes(fileName), device) { }
        /// a compact key blob (SaveCompactKeys, magic "CNHK") is recognised too: its keys are expanded on the GPU, there is no secret key
        public B200BfvFactory(byte[] archive, int device = 0)
        {
            bool compact = archive.Length >= 4 && archive[0] == (byte)'C' && archive[1] == (byte)'N' && archive[2] == (byte)'H' && archive[3] == (byte)'K';
            if (compact) Cnhe.Check(Cnhe.cnhe_context_load_compact(archive, (UIntPtr)archive.Length, device, out Ctx));
            else Cnhe.Check(Cnhe.cnhe_context_load(archive, (UIntPtr)archive.Length, device, out Ctx));
            Cnhe.Check(Cnhe.cnhe_context_info(Ctx, out _, out _, out int P, out _, out _, out _));
            var primes = new ulong[P];
            Cnhe.Check(Cnhe.cnhe_context_plain_moduli(Ctx, primes));
            env = new B200BfvEnvironment { ParentFactory = this };
            SetPrimes(primes);
        }
        void SetPrimes(ulong[] primes)
        {
            Primes = primes;
            BigFactor = primes.Aggregate(BigInteger.One, (a, p) => a * p);
            PreComputedCoefficients = primes.Select(p =>
            {
                var minor = BigFactor / p;
                return minor * BigInteger.ModPow(minor % p, p - 2, p); // inverse modulo the prime p
            }).ToArray();
        }

        public IComputationEnvironment AllocateComputationEnv() => env;
        public void FreeComputationEnv(IComputationEnvironment e) { }

        IVector Make(Vector<double> v, EVectorFormat format, double scale, bool encrypt)
        {
            var a = v.ToArray();
            IntPtr h;
            Cnhe.Check(encrypt ? Cnhe.cnhe_vec_encrypt(Ctx, a, (ulong)a.Length, scale, (int)format, out h)
                               : Cnhe.cnhe_vec_plain(Ctx, a, (ulong)a.Length, scale, (int)format, out h));
            return new B200BfvVector(this, h);
        }
        IVector MakeBig(IEnumerable<BigInteger> v, EVectorFormat format, bool encrypt)
        {   // SplitBigNumbers(IEnumerable<BigInteger>) (EncryptedSealBfvVector.cs:367-379)
            var vals = v.Select(x => ((x % BigFactor) + BigFactor) % BigFactor).ToArray();
            var res = new ulong[vals.Length * Primes.Length];
            for (int i = 0; i < Primes.Length; i++)
                for (int j = 0; j < vals.Length; j++) res[i * vals.Length + j] = (ulong)(vals[j] % Primes[i]);
            Cnhe.Check(Cnhe.cnhe_vec_from_residues(Ctx, res, (ulong)vals.Length, 1.0, (int)format, encrypt ? 1 : 0, out var h));
            return new B200BfvVector(this, h);
        }
        public IVector GetPlainVector(Vector<double> v, EVectorFormat format, double scale) => Make(v, format, scale, false);
        public IVector GetPlainVector(IEnumerable<BigInteger> v, EVectorFormat format) => MakeBig(v, format, false);
        public IVector GetEncryptedVector(Vector<double> v, EVectorFormat format, double scale) => Make(v, format, scale, true);
        public IVector GetEncryptedVector(IEnumerable<BigInteger> v, EVectorFormat format) => MakeBig(v, format, true);
        public IVector CopyVector(IVector v)
        {
            Cnhe.Check(Cnhe.cnhe_vec_copy(Ctx, ((B200BfvVector)v).Handle, out var h));
            return new B200BfvVector(this, h);
        }
        public BigInteger GetValueFromString(string str)
        {   // IFactory.cs:395-403
            var f = str.Split(',').Select(BigInteger.Parse).ToArray();
            BigInteger x = 0;
            for (int i = 0; i < f.Length; i++) x += PreComputedCoefficients[i] * f[i];
            return x % BigFactor;
        }
        public string GetStringFromValue(BigInteger value) => string.Join(",", Primes.Select(p => (((value % p) + p) % p).ToString())); // IFactory.cs:405-409

        public IMatrix GetPlainMatrix(Matrix<double> m, EMatrixFormat format, double scale)
        {   // IFactory.cs:330-351
            var vecs = (format == EMatrixFormat.ColumnMajor ? m.EnumerateColumns() : m.EnumerateRows())
                .Select(v => GetPlainVector(v, EVectorFormat.dense, scale)).ToArray();
            return new B200BfvMatrix(this, vecs, format, false) { DataDisposedExternaly = false };
        }
        public IMatrix GetEncryptedMatrix(Matrix<double> m, EMatrixFormat format, double scale)
        {   // IFactory.cs:353-380, one encryption wave for the whole matrix
            var rows = (format == EMatrixFormat.ColumnMajor ? m.EnumerateColumns() : m.EnumerateRows()).ToArray();
            ulong dim = (ulong)rows[0].Count;
            var flat = rows.SelectMany(r => r.ToArray()).ToArray();
            var hs = new IntPtr[rows.Length];
            Cnhe.Check(Cnhe.cnhe_vecs_encrypt(Ctx, flat, rows.Length, dim, scale, hs));
            return new B200BfvMatrix(this, hs.Select(h => (IVector)new B200BfvVector(this, h)).ToArray(), format, false) { DataDisposedExternaly = false };
        }
        // the same encryption as one compact blob (bit-packed c0, per-channel ChaCha20 keys for c1; include/cnhe.h); needs the secret key
        public byte[] GetEncryptedMatrixCompact(Matrix<double> m, EMatrixFormat format, double scale)
        {
            var rows = (format == EMatrixFormat.ColumnMajor ? m.EnumerateColumns() : m.EnumerateRows()).ToArray();
            ulong dim = (ulong)rows[0].Count;
            var flat = rows.SelectMany(r => r.ToArray()).ToArray();
            Cnhe.Check(Cnhe.cnhe_vecs_encrypt_compact(Ctx, flat, rows.Length, dim, scale, null, UIntPtr.Zero, out UIntPtr needed));
            var blob = new byte[(long)needed.ToUInt64()];
            Cnhe.Check(Cnhe.cnhe_vecs_encrypt_compact(Ctx, flat, rows.Length, dim, scale, blob, needed, out needed));
            return blob;
        }
        // the matrix of a compact blob, expanded on the GPU; the format travels out of band (as with raw import)
        public IMatrix LoadCompactMatrix(byte[] data, EMatrixFormat format)
        {
            int cap = BitConverter.ToInt32(data, 20); // header field n
            var hs = new IntPtr[Math.Max(cap, 1)];
            Cnhe.Check(Cnhe.cnhe_vecs_import_compact(Ctx, data, (UIntPtr)(ulong)data.Length, hs, cap, out int n));
            return new B200BfvMatrix(this, hs.Take(n).Select(h => (IVector)new B200BfvVector(this, h)).ToArray(), format, false) { DataDisposedExternaly = false };
        }
        public IMatrix GetMatrix(IVector[] vectors, EMatrixFormat format, bool CopyVectors = true) => new B200BfvMatrix(this, vectors, format, CopyVectors);

        static string ReadBlock(StreamReader str, string endMarker)
        {
            var sb = new StringBuilder();
            while (true)
            {
                var line = str.ReadLine();
                if (line == null) throw new Exception("Bad stream format.");
                sb.Append(line).Append("\n");
                if (line == endMarker) return sb.ToString();
            }
        }
        public IVector LoadVector(StreamReader str)
        {   // IFactory.cs:479-483 -> EncryptedSealBfvVector.Read (:414-427)
            var text = Encoding.ASCII.GetBytes(ReadBlock(str, "<End LargeEncryptedVector>"));
            Cnhe.Check(Cnhe.cnhe_vec_read(Ctx, text, (UIntPtr)text.Length, out var h, out _));
            return new B200BfvVector(this, h);
        }
        public IMatrix LoadMatrix(StreamReader str)
        {   // IFactory.cs:474-478 -> EncryptedSealBfvMatrix.Read (:182-197)
            if (str.ReadLine() != "<Start LargeEncryptedMatrix>") throw new Exception("Bad stream format.");
            var format = (EMatrixFormat)Enum.Parse(typeof(EMatrixFormat), str.ReadLine());
            var vecs = new IVector[int.Parse(str.ReadLine())];
            for (int i = 0; i < vecs.Length; i++) vecs[i] = LoadVector(str);
            if (str.ReadLine() != "<End LargeEncryptedMatrix>") throw new Exception("Bad stream format.");
            return new B200BfvMatrix(this, vecs, format, false) { DataDisposedExternaly = false };
        }
        public Stream Save(Stream stream, bool withPrivateKeys = false)
        {   // IFactory.cs:484-488 -> EncryptedSealBfvEnvironment.Save (EncryptedSealBfvVector.cs:104-126)
            Cnhe.Check(Cnhe.cnhe_keys_save(Ctx, withPrivateKeys ? 1 : 0, null, UIntPtr.Zero, out var needed));
            var buf = new byte[(long)needed];
            Cnhe.Check(Cnhe.cnhe_keys_save(Ctx, withPrivateKeys ? 1 : 0, buf, needed, out needed));
            stream.Write(buf, 0, buf.Length);
            return stream;
        }
        public void Save(string FileName, bool withPrivateKeys = false)
        {
            using (var f = new FileStream(FileName, FileMode.Create)) { Save(f, withPrivateKeys); f.Flush(); }
        }
        /// the evaluation keys a server needs as one compact blob (include/cnhe.h, cnhe_keys_save_compact): a fresh key set under this
        /// factory's secret key; galois null = every standard element, empty = none, else the elements the network rotates by
        public byte[] SaveCompactKeys(bool publicKey = true, bool relin = true, ulong[] galois = null)
        {
            int sets = (publicKey ? 1 : 0) | (relin ? 2 : 0), n = galois == null ? -1 : galois.Length;
            Cnhe.Check(Cnhe.cnhe_keys_save_compact(Ctx, sets, galois, n, null, UIntPtr.Zero, out var needed));
            var buf = new byte[(long)needed];
            Cnhe.Check(Cnhe.cnhe_keys_save_compact(Ctx, sets, galois, n, buf, needed, out needed));
            return buf;
        }

        /// fused PoolLayer.Apply (NeuralNetworks/PoolLayer.cs:149-229): one device call for the whole layer instead of the per-output fan-out
        public IVector[] ConvDenseLayer(IVector[] inputs, int[] gather, IVector[] weights, IVector[] bias, int M, int K)
        {
            var outs = new IntPtr[M];
            Cnhe.Check(Cnhe.cnhe_layer_conv_dense(Ctx, Cnhe.Handles(inputs), inputs.Length, gather, Cnhe.Handles(weights), bias == null ? null : Cnhe.Handles(bias),
                                                  M, K, outs));
            return outs.Select(h => (IVector)new B200BfvVector(this, h)).ToArray();
        }
        /// SquareActivation.Apply (NeuralNetworks/SquareActivation.cs:10-13) over every column in one wave
        public IVector[] SquareLayer(IVector[] inputs)
        {
            var outs = new IntPtr[inputs.Length];
            Cnhe.Check(Cnhe.cnhe_layer_square(Ctx, Cnhe.Handles(inputs), inputs.Length, outs));
            return outs.Select(h => (IVector)new B200BfvVector(this, h)).ToArray();
        }
        /// Records the library calls `record` makes (one inference through the layers after the EncryptLayer, on example inputs) as one CUDA
        /// graph instead of running them (include/cnhe.h, cnhe_capture_begin).  Returns the graph; the vectors `record` created belong to it.
        /// A call that cannot be recorded (decryption, encryption, a synchronising timer) throws and aborts the recording.
        public IntPtr Capture(Action record)
        {
            Cnhe.Check(Cnhe.cnhe_capture_begin(Ctx));
            try { record(); }
            catch { Cnhe.cnhe_capture_abort(Ctx); throw; }
            Cnhe.Check(Cnhe.cnhe_capture_end(Ctx, out var graph));
            return graph;
        }
        /// Capture of a levelled inference: `levels` are the contexts (cnhe_context_derive_level of this factory's) its mod switches go to.
        /// Their calls and the switches between them are recorded into the same graph (include/cnhe.h, cnhe_capture_begin_levels); the
        /// graph must be disposed before any of those contexts.
        public IntPtr CaptureLevels(IntPtr[] levels, Action record)
        {
            Cnhe.Check(Cnhe.cnhe_capture_begin_levels(Ctx, levels, levels.Length));
            try { record(); }
            catch { Cnhe.cnhe_capture_abort(Ctx); throw; }
            Cnhe.Check(Cnhe.cnhe_capture_end(Ctx, out var graph));
            return graph;
        }
        /// One replay of a Capture graph: `inputs` are copied into the vectors the recording read as its inputs (same shapes and scales),
        /// then the graph is launched.  The inputs may belong to other clients (key slots) than the recorded ones: the graph is bound to
        /// their slots first (include/cnhe.h, cnhe_graph_bind), and the recorded inputs and outputs report them.  The slots the recorded
        /// inputs carry at a graph's first Run are taken as the ones it was recorded in.  The recorded outputs hold this run's words until
        /// the next Run.
        public void Run(IntPtr graph, IVector[] recordedInputs, IVector[] inputs)
        {
            if (recordedInputs.Length != inputs.Length) throw new Exception("the inputs are not shaped as the recorded ones");
            IntPtr[] dst = Cnhe.Handles(recordedInputs), src = Cnhe.Handles(inputs);
            if (!recordedSlots.TryGetValue(graph, out var recorded))
                recordedSlots[graph] = recorded = dst.Select(KeySlot).ToArray();
            int[] current = src.Select(KeySlot).ToArray();
            Cnhe.Check(Cnhe.cnhe_graph_bind(graph, GraphBinding(graph, recorded, current), GraphSlots(graph).Length));
            for (int i = 0; i < dst.Length; i++)
                if (KeySlot(dst[i]) != current[i]) Cnhe.Check(Cnhe.cnhe_vec_set_key_slot(dst[i], current[i]));
            Cnhe.Check(Cnhe.cnhe_vecs_assign(Ctx, dst, src, inputs.Length));
            Cnhe.Check(Cnhe.cnhe_graph_launch(graph));
        }
        readonly Dictionary<IntPtr, int[]> recordedSlots = new Dictionary<IntPtr, int[]>();
        static int KeySlot(IntPtr v) { Cnhe.Check(Cnhe.cnhe_vec_key_slot(v, out int s)); return s; }
        static int[] GraphSlots(IntPtr graph)
        {
            Cnhe.Check(Cnhe.cnhe_graph_slots(graph, null, 0, out int n));
            var slots = new int[n];
            Cnhe.Check(Cnhe.cnhe_graph_slots(graph, slots, n, out n));
            return slots;
        }
        /// The slot each key position of `graph` is bound to when recorded input j (recorded in slot recorded[j]) takes an input of slot
        /// current[j]; a position no input was recorded in keeps its own slot.  Throws, before anything changes, when one recorded slot would
        /// be bound to two slots.
        static int[] GraphBinding(IntPtr graph, int[] recorded, int[] current)
        {
            var to = new Dictionary<int, int>();
            for (int j = 0; j < recorded.Length; j++)
            {
                if (to.TryGetValue(recorded[j], out int c) && c != current[j])
                    throw new Exception($"the inputs bind recorded key slot {recorded[j]} to two key slots ({c} and {current[j]})");
                to[recorded[j]] = current[j];
            }
            return GraphSlots(graph).Select(p => to.TryGetValue(p, out int s) ? s : p).ToArray();
        }
        public void DisposeCapture(IntPtr graph)
        {
            recordedSlots.Remove(graph);
            Cnhe.Check(Cnhe.cnhe_graph_destroy(graph));
        }
        /// CryptoTracker.TestBudget (CryptoTracker.cs:41-52)
        public int NoiseBudget(IVector v, int channel = 0, int block = 0)
        {
            Cnhe.Check(Cnhe.cnhe_noise_budget(Ctx, ((B200BfvVector)v).Handle, channel, block, out int bits));
            return bits;
        }
        public void Dispose()
        {
            if (Ctx != IntPtr.Zero) { Cnhe.cnhe_context_destroy(Ctx); Ctx = IntPtr.Zero; }
        }
    }
}
