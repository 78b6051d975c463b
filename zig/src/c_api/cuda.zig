//! CUDA propagation library bindings -- GENERATED from include/astroz_b200.h by tools/gen_zig_bindings.py.
//! Drop this file in as src/c_api/cuda.zig of ATTron/astroz (next to src/c_api/sgp4.zig); INTEGRATION.md has
//! the build.zig wiring and zig/src/Constellation.device.zig the device branch of Constellation.zig.
//! Error codes are err.Code values (src/c_api/error.zig:3-19) extended with cudaError = -200, noCudaDevice = -201.
//! Uncompiled here: the build image has no Zig toolchain (DESIGN.md section 1).

pub const Handle = ?*anyopaque;

pub const astroz_force_model_t = extern struct {
    kind: i32,
    flags: u32,
    mu: f64,
    coef: f64,
    r_eq: f64,
    rho0: f64,
    scale_height: f64,
    max_altitude: f64,
    f107: f64,
    c: f64,
    area: f64,
    mass: f64,
    pos: [3]f64,
    c_per_state: ?[*]const f64,
    area_per_state: ?[*]const f64,
    mass_per_state: ?[*]const f64,
    pos_table: ?[*]const f64,
};

pub const astroz_impulse_t = extern struct {
    time: f64,
    kind: i32,
    reserved: u32,
    p: [3]f64,
};

pub extern fn astroz_cuda_version() u32;
pub extern fn astroz_cuda_device_count() i32;
pub extern fn astroz_cuda_last_error() [*:0]const u8;
pub extern fn astroz_cuda_host_alloc(bytes: usize) ?*anyopaque;
pub extern fn astroz_cuda_host_free(p: ?*anyopaque) void;
pub extern fn astroz_cuda_host_register(p: ?*anyopaque, bytes: usize) i32;
pub extern fn astroz_cuda_host_unregister(p: ?*anyopaque) i32;
pub extern fn astroz_cuda_constellation_create(line1: [*]const [*:0]const u8, line2: [*]const [*:0]const u8, n: u32, grav: i32, device: i32, out: *Handle) i32;
pub extern fn astroz_cuda_constellation_create_from_text(text: [*]const u8, len: usize, grav: i32, device: i32, out: *Handle) i32;
pub extern fn astroz_cuda_constellation_create_from_elements(epoch_jd: ?[*]const f64, mean_motion_rev_day: ?[*]const f64, ecc: ?[*]const f64, incl_deg: ?[*]const f64, raan_deg: ?[*]const f64, argp_deg: ?[*]const f64, ma_deg: ?[*]const f64, bstar: ?[*]const f64, n: u32, grav: i32, device: i32, out: *Handle) i32;
pub extern fn astroz_cuda_constellation_create_from_elements_device(d_epoch_jd: ?[*]const f64, d_mean_motion_rev_day: ?[*]const f64, d_ecc: ?[*]const f64, d_incl_deg: ?[*]const f64, d_raan_deg: ?[*]const f64, d_argp_deg: ?[*]const f64, d_ma_deg: ?[*]const f64, d_bstar: ?[*]const f64, n: u32, grav: i32, device: i32, out: *Handle) i32;
pub extern fn astroz_cuda_constellation_free(h: Handle) void;
pub extern fn astroz_cuda_constellation_counts(h: Handle, n: ?[*]u32, n_sgp4: ?[*]u32, n_sdp4: ?[*]u32) i32;
pub extern fn astroz_cuda_constellation_epochs(h: Handle, epochs: ?[*]f64) i32;
pub extern fn astroz_cuda_constellation_classes(h: Handle, classes: ?[*]i32) i32;
pub extern fn astroz_cuda_constellation_get_reference_epoch(h: Handle, jd: ?[*]f64) i32;
pub extern fn astroz_cuda_constellation_set_reference_epoch(h: Handle, jd: f64) i32;
pub extern fn astroz_cuda_constellation_propagate(h: Handle, jd: ?[*]const f64, fr: ?[*]const f64, n_times: u32, pos: ?[*]f64, vel: ?[*]f64, mode: i32, layout: i32) i32;
pub extern fn astroz_cuda_constellation_propagate_device(h: Handle, jd: ?[*]const f64, fr: ?[*]const f64, n_times: u32, d_pos: ?[*]f64, d_vel: ?[*]f64, d_status: ?[*]u8, mode: i32, layout: i32, out_num_sats: u32, out_sat_offset: u32, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_constellation_propagate_pairs(h: Handle, sat: ?[*]const u32, jd: ?[*]const f64, fr: ?[*]const f64, n: u32, mode: i32, pos: ?[*]f64, vel: ?[*]f64, status: ?[*]u8) i32;
pub extern fn astroz_cuda_constellation_propagate_pairs_device(h: Handle, d_sat: ?[*]const u32, d_jd: ?[*]const f64, d_fr: ?[*]const f64, n: u32, mode: i32, d_pos: ?[*]f64, d_vel: ?[*]f64, d_status: ?[*]u8, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_constellation_propagate_gather(h: Handle, jd: ?[*]const f64, fr: ?[*]const f64, n_times: u32, peer_pos: ?[*]const ?*anyopaque, peer_vel: ?[*]const ?*anyopaque, n_peers: u32, mc_pos: ?*anyopaque, mc_vel: ?*anyopaque, out_num_sats: u32, out_sat_offset: u32, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_constellation_host_block(h: Handle, n_times: u32, layout: i32, out: ?[*]?[*]f64) i32;
pub extern fn astroz_cuda_constellation_devices(h: Handle, n_devices: ?[*]i32, device_ids: ?[*]i32, first_rows: ?[*]u32) i32;
pub extern fn astroz_cuda_constellation_propagate_replicated(h: Handle, jd: ?[*]const f64, fr: ?[*]const f64, n_times: u32, velocities: i32, d_pos: ?[*]?[*]f64, d_vel: ?[*]?[*]f64) i32;
pub extern fn astroz_cuda_constellation_reset_carry(h: Handle) i32;
pub extern fn astroz_cuda_sgp4_propagate_into(h: Handle, times: ?[*]const f64, n_times: u32, epoch_offsets: ?[*]const f64, pos: ?[*]f64, vel: ?[*]f64, mode: i32, reference_jd: f64, layout: i32, satellite_mask: ?[*]const u8, out_num_sats: u32) i32;
pub extern fn astroz_cuda_sgp4_propagate_into_device(h: Handle, times: ?[*]const f64, n_times: u32, epoch_offsets: ?[*]const f64, d_pos: ?[*]f64, d_vel: ?[*]f64, mode: i32, reference_jd: f64, layout: i32, satellite_mask: ?[*]const u8, out_num_sats: u32, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_sdp4_propagate_into(h: Handle, jd: ?[*]const f64, fr: ?[*]const f64, n_times: u32, pos: ?[*]f64, vel: ?[*]f64, mode: i32, layout: i32, out_num_sats: u32, sat_offset: u32) i32;
pub extern fn astroz_cuda_sdp4_propagate_into_device(h: Handle, jd: ?[*]const f64, fr: ?[*]const f64, n_times: u32, d_pos: ?[*]f64, d_vel: ?[*]f64, mode: i32, layout: i32, out_num_sats: u32, sat_offset: u32, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_sgp4_screen(h: Handle, times: ?[*]const f64, n_times: u32, epoch_offsets: ?[*]const f64, target_idx: u32, threshold: f64, reference_jd: f64, out_min_dists: ?[*]f64, out_min_t: ?[*]u32) i32;
pub extern fn astroz_cuda_constellation_coarse_screen_device(h: Handle, d_positions: ?[*]const f64, num_sats: u32, num_times: u32, layout: i32, threshold: f64, d_valid_mask: ?[*]const u8, d_pairs: ?[*]u32, d_t_indices: ?[*]u32, max_results: u32, count: *u64) i32;
pub extern fn astroz_cuda_sgp4_screen_all(h: Handle, times: ?[*]const f64, n_times: u32, epoch_offsets: ?[*]const f64, threshold: f64, pairs: ?[*]u32, t_indices: ?[*]u32, max_results: u32, count: *u64) i32;
pub extern fn astroz_cuda_constellation_synchronize(h: Handle) i32;
pub extern fn astroz_cuda_constellation_set_timing(h: Handle, enabled: i32) i32;
pub extern fn astroz_cuda_constellation_last_kernel_ms(h: Handle, ms: *[3]f32) i32;
pub extern fn astroz_cuda_sgp4_init(line1: [*:0]const u8, line2: [*:0]const u8, grav: i32, device: i32, out: *Handle) i32;
pub extern fn astroz_cuda_sgp4_free(h: Handle) void;
pub extern fn astroz_cuda_sgp4_is_deep_space(h: Handle) i32;
pub extern fn astroz_cuda_sgp4_epoch(h: Handle, epoch_jd: ?[*]f64) i32;
pub extern fn astroz_cuda_sgp4_elements(h: Handle, out10: ?[*]f64) i32;
pub extern fn astroz_cuda_sgp4_propagate(h: Handle, tsince: f64, pos: *[3]f64, vel: *[3]f64) i32;
pub extern fn astroz_cuda_sgp4_propagate_batch(h: Handle, times: ?[*]const f64, results: ?[*]f64, count: u32) i32;
pub extern fn astroz_cuda_sgp4_array(h: Handle, jd: ?[*]const f64, fr: ?[*]const f64, epoch_jd: f64, results: ?[*]f64, count: u32) i32;
pub extern fn astroz_cuda_constellation_propagate_device_f32(h: Handle, jd: ?[*]const f64, fr: ?[*]const f64, n_times: u32, d_pos: ?[*]f64, d_vel: ?[*]f64, phase64: i32, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_numerical_times(t0: f64, duration: f64, dt: f64, times: ?[*]f64, count: *u64) i32;
pub extern fn astroz_cuda_propagate_numerical(states: ?[*]const f64, n: u32, t0: f64, duration: f64, dt: f64, mu: f64, forces: i32, j2: ?[*]const f64, r_eq: ?[*]const f64, drag_cd: ?[*]const f64, drag_area: ?[*]const f64, drag_mass: ?[*]const f64, integrator: i32, rtol: f64, atol: f64, device: i32, out: ?[*]f64, status: ?[*]u8, steps: ?[*]u64) i32;
pub extern fn astroz_cuda_propagate_numerical_device(d_states: ?[*]const f64, n: u32, t0: f64, duration: f64, dt: f64, mu: f64, forces: i32, j2: ?[*]const f64, r_eq: ?[*]const f64, d_drag_cd: ?[*]const f64, d_drag_area: ?[*]const f64, d_drag_mass: ?[*]const f64, integrator: i32, rtol: f64, atol: f64, device: i32, d_out: ?[*]f64, d_status: ?[*]u8, d_steps: ?[*]u64, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_propagate_numerical_models(states: ?[*]const f64, n: u32, t0: f64, duration: f64, dt: f64, models: ?[*]const astroz_force_model_t, n_models: u32, integrator: i32, rtol: f64, atol: f64, device: i32, out: ?[*]f64, status: ?[*]u8, steps: ?[*]u64) i32;
pub extern fn astroz_cuda_propagate_numerical_models_device(d_states: ?[*]const f64, n: u32, t0: f64, duration: f64, dt: f64, models: ?[*]const astroz_force_model_t, n_models: u32, integrator: i32, rtol: f64, atol: f64, device: i32, d_out: ?[*]f64, d_status: ?[*]u8, d_steps: ?[*]u64, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_propagate_maneuvers(states: ?[*]const f64, n: u32, t0: f64, duration: f64, h: f64, mu: f64, impulse_offsets: ?[*]const u32, impulses: ?[*]const astroz_impulse_t, m: u32, models: ?[*]const astroz_force_model_t, n_models: u32, integrator: i32, rtol: f64, atol: f64, max_samples: u32, device: i32, times: ?[*]f64, out: ?[*]f64, n_samples: ?[*]u64, status: ?[*]u8, steps: ?[*]u64) i32;
pub extern fn astroz_cuda_propagate_maneuvers_device(d_states: ?[*]const f64, n: u32, t0: f64, duration: f64, h: f64, mu: f64, d_impulse_offsets: ?[*]const u32, d_impulses: ?[*]const astroz_impulse_t, m: u32, models: ?[*]const astroz_force_model_t, n_models: u32, integrator: i32, rtol: f64, atol: f64, max_samples: u32, device: i32, d_times: ?[*]f64, d_out: ?[*]f64, d_n_samples: ?[*]u64, d_status: ?[*]u8, d_steps: ?[*]u64, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_fit_elements(elements: ?[*]const f64, n: u32, grav: i32, offsets: ?[*]const u32, jd: ?[*]const f64, fr: ?[*]const f64, pos: ?[*]const f64, vel: ?[*]const f64, m: u32, pos_sigma: f64, vel_sigma: f64, fit_bstar: i32, max_iter: u32, device: i32, fitted: ?[*]f64, rms: ?[*]f64, iterations: ?[*]u32, status: ?[*]u8) i32;
pub extern fn astroz_cuda_fit_elements_device(d_elements: ?[*]const f64, n: u32, grav: i32, d_offsets: ?[*]const u32, d_jd: ?[*]const f64, d_fr: ?[*]const f64, d_pos: ?[*]const f64, d_vel: ?[*]const f64, pos_sigma: f64, vel_sigma: f64, fit_bstar: i32, max_iter: u32, device: i32, d_fitted: ?[*]f64, d_rms: ?[*]f64, d_iterations: ?[*]u32, d_status: ?[*]u8, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_fit_elements_mixed(elements: ?[*]const f64, n: u32, grav: i32, offsets: ?[*]const u32, jd: ?[*]const f64, fr: ?[*]const f64, pos: ?[*]const f64, vel: ?[*]const f64, m: u32, pos_sigma: f64, vel_sigma: f64, fit_bstar: i32, max_iter: u32, device: i32, fitted: ?[*]f64, rms: ?[*]f64, iterations: ?[*]u32, status: ?[*]u8) i32;
pub extern fn astroz_cuda_fit_elements_mixed_device(d_elements: ?[*]const f64, n: u32, grav: i32, d_offsets: ?[*]const u32, d_jd: ?[*]const f64, d_fr: ?[*]const f64, d_pos: ?[*]const f64, d_vel: ?[*]const f64, pos_sigma: f64, vel_sigma: f64, fit_bstar: i32, max_iter: u32, device: i32, d_fitted: ?[*]f64, d_rms: ?[*]f64, d_iterations: ?[*]u32, d_status: ?[*]u8, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_fit_observations(elements: ?[*]const f64, n: u32, grav: i32, offsets: ?[*]const u32, jd: ?[*]const f64, fr: ?[*]const f64, value: ?[*]const f64, sigma: ?[*]const f64, station: ?[*]const u32, kind: ?[*]const u8, m: u32, stations: ?[*]const f64, k: u32, fit_bstar: i32, max_iter: u32, device: i32, fitted: ?[*]f64, wrms: ?[*]f64, n_residuals: ?[*]u32, covariance: ?[*]f64, iterations: ?[*]u32, status: ?[*]u8, model: ?[*]u8) i32;
pub extern fn astroz_cuda_fit_observations_mixed(elements: ?[*]const f64, n: u32, grav: i32, offsets: ?[*]const u32, jd: ?[*]const f64, fr: ?[*]const f64, value: ?[*]const f64, sigma: ?[*]const f64, station: ?[*]const u32, kind: ?[*]const u8, m: u32, stations: ?[*]const f64, k: u32, fit_bstar: i32, max_iter: u32, device: i32, fitted: ?[*]f64, wrms: ?[*]f64, n_residuals: ?[*]u32, covariance: ?[*]f64, iterations: ?[*]u32, status: ?[*]u8, model: ?[*]u8) i32;
pub extern fn astroz_cuda_fit_observations_device(d_elements: ?[*]const f64, n: u32, grav: i32, d_offsets: ?[*]const u32, d_jd: ?[*]const f64, d_fr: ?[*]const f64, d_value: ?[*]const f64, d_sigma: ?[*]const f64, d_station: ?[*]const u32, d_kind: ?[*]const u8, d_stations: ?[*]const f64, fit_bstar: i32, max_iter: u32, device: i32, d_fitted: ?[*]f64, d_wrms: ?[*]f64, d_n_residuals: ?[*]u32, d_covariance: ?[*]f64, d_iterations: ?[*]u32, d_status: ?[*]u8, d_model: ?[*]u8, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_fit_observations_mixed_device(d_elements: ?[*]const f64, n: u32, grav: i32, d_offsets: ?[*]const u32, d_jd: ?[*]const f64, d_fr: ?[*]const f64, d_value: ?[*]const f64, d_sigma: ?[*]const f64, d_station: ?[*]const u32, d_kind: ?[*]const u8, d_stations: ?[*]const f64, fit_bstar: i32, max_iter: u32, device: i32, d_fitted: ?[*]f64, d_wrms: ?[*]f64, d_n_residuals: ?[*]u32, d_covariance: ?[*]f64, d_iterations: ?[*]u32, d_status: ?[*]u8, d_model: ?[*]u8, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_observe(states: ?[*]const f64, jd: ?[*]const f64, fr: ?[*]const f64, kind: ?[*]const u8, station: ?[*]const u32, m: u32, stations: ?[*]const f64, k: u32, device: i32, values: ?[*]f64) i32;
pub extern fn astroz_cuda_observe_device(d_states: ?[*]const f64, d_jd: ?[*]const f64, d_fr: ?[*]const f64, d_kind: ?[*]const u8, d_station: ?[*]const u32, m: u32, d_stations: ?[*]const f64, device: i32, d_values: ?[*]f64, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_propagate_covariance(elements: ?[*]const f64, n: u32, grav: i32, covariance: ?[*]const f64, model: ?[*]const u8, offsets: ?[*]const u32, jd: ?[*]const f64, fr: ?[*]const f64, m: u32, frame: i32, device: i32, state: ?[*]f64, state_covariance: ?[*]f64, jacobian: ?[*]f64, status: ?[*]u8) i32;
pub extern fn astroz_cuda_propagate_covariance_device(d_elements: ?[*]const f64, n: u32, grav: i32, d_covariance: ?[*]const f64, d_model: ?[*]const u8, d_offsets: ?[*]const u32, d_jd: ?[*]const f64, d_fr: ?[*]const f64, m: u32, frame: i32, device: i32, d_state: ?[*]f64, d_state_covariance: ?[*]f64, d_jacobian: ?[*]f64, d_status: ?[*]u8, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_conjunction(elements: ?[*]const f64, n: u32, grav: i32, covariance: ?[*]const f64, model: ?[*]const u8, primary: ?[*]const u32, secondary: ?[*]const u32, jd: ?[*]const f64, fr: ?[*]const f64, window_min: ?[*]const f64, hbr_km: ?[*]const f64, m: u32, frame: i32, device: i32, record: ?[*]f64, states: ?[*]f64, state_covariance: ?[*]f64, status: ?[*]u8) i32;
pub extern fn astroz_cuda_conjunction_device(d_elements: ?[*]const f64, n: u32, grav: i32, d_covariance: ?[*]const f64, d_model: ?[*]const u8, d_primary: ?[*]const u32, d_secondary: ?[*]const u32, d_jd: ?[*]const f64, d_fr: ?[*]const f64, d_window_min: ?[*]const f64, d_hbr_km: ?[*]const f64, m: u32, frame: i32, device: i32, d_record: ?[*]f64, d_states: ?[*]f64, d_state_covariance: ?[*]f64, d_status: ?[*]u8, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_conjunction_mc(elements: ?[*]const f64, n: u32, grav: i32, covariance: ?[*]const f64, model: ?[*]const u8, primary: ?[*]const u32, secondary: ?[*]const u32, jd: ?[*]const f64, fr: ?[*]const f64, window_min: ?[*]const f64, hbr_km: ?[*]const f64, samples: ?[*]const u64, first: ?[*]const u64, seed: ?[*]const u64, m: u32, record: u32, device: i32, counts: ?[*]u64, sample_out: ?[*]f64, status: ?[*]u8) i32;
pub extern fn astroz_cuda_conjunction_mc_device(d_elements: ?[*]const f64, n: u32, grav: i32, d_covariance: ?[*]const f64, d_model: ?[*]const u8, d_primary: ?[*]const u32, d_secondary: ?[*]const u32, d_jd: ?[*]const f64, d_fr: ?[*]const f64, d_window_min: ?[*]const f64, d_hbr_km: ?[*]const f64, d_samples: ?[*]const u64, d_first: ?[*]const u64, d_seed: ?[*]const u64, m: u32, record: u32, device: i32, d_counts: ?[*]u64, d_sample_out: ?[*]f64, d_status: ?[*]u8, d_scratch: ?*anyopaque, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_conjunction_mc_scratch_bytes(m: u32, bytes: *u64) i32;
pub extern fn astroz_cuda_conjunction_is(elements: ?[*]const f64, n: u32, grav: i32, covariance: ?[*]const f64, model: ?[*]const u8, primary: ?[*]const u32, secondary: ?[*]const u32, jd: ?[*]const f64, fr: ?[*]const f64, window_min: ?[*]const f64, hbr_km: ?[*]const f64, samples: ?[*]const u64, first: ?[*]const u64, seed: ?[*]const u64, shift: ?[*]const f64, m: u32, record: u32, device: i32, counts: ?[*]u64, proposal: ?[*]f64, proposal_kind: ?[*]u8, sample_out: ?[*]f64, status: ?[*]u8) i32;
pub extern fn astroz_cuda_conjunction_is_device(d_elements: ?[*]const f64, n: u32, grav: i32, d_covariance: ?[*]const f64, d_model: ?[*]const u8, d_primary: ?[*]const u32, d_secondary: ?[*]const u32, d_jd: ?[*]const f64, d_fr: ?[*]const f64, d_window_min: ?[*]const f64, d_hbr_km: ?[*]const f64, d_samples: ?[*]const u64, d_first: ?[*]const u64, d_seed: ?[*]const u64, d_shift: ?[*]const f64, m: u32, record: u32, device: i32, d_counts: ?[*]u64, d_proposal: ?[*]f64, d_proposal_kind: ?[*]u8, d_sample_out: ?[*]f64, d_status: ?[*]u8, d_scratch: ?*anyopaque, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_conjunction_is_scratch_bytes(m: u32, bytes: *u64) i32;
pub extern fn astroz_cuda_conjunction_maneuver(elements: ?[*]const f64, n: u32, grav: i32, covariance: ?[*]const f64, model: ?[*]const u8, primary: ?[*]const u32, secondary: ?[*]const u32, jd: ?[*]const f64, fr: ?[*]const f64, window_min: ?[*]const f64, hbr_km: ?[*]const f64, m: u32, candidate: ?[*]const u32, burn_jd: ?[*]const f64, burn_fr: ?[*]const f64, dv_rtn: ?[*]const f64, dv_sigma: ?[*]const f64, t: u32, device: i32, record: ?[*]f64, new_elements: ?[*]f64, new_covariance: ?[*]f64, residual: ?[*]f64, status: ?[*]u8) i32;
pub extern fn astroz_cuda_conjunction_maneuver_device(d_elements: ?[*]const f64, n: u32, grav: i32, d_covariance: ?[*]const f64, d_model: ?[*]const u8, d_primary: ?[*]const u32, d_secondary: ?[*]const u32, d_jd: ?[*]const f64, d_fr: ?[*]const f64, d_window_min: ?[*]const f64, d_hbr_km: ?[*]const f64, m: u32, d_candidate: ?[*]const u32, d_burn_jd: ?[*]const f64, d_burn_fr: ?[*]const f64, d_dv_rtn: ?[*]const f64, d_dv_sigma: ?[*]const f64, t: u32, device: i32, d_record: ?[*]f64, d_new_elements: ?[*]f64, d_new_covariance: ?[*]f64, d_residual: ?[*]f64, d_status: ?[*]u8, d_scratch: ?*anyopaque, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_conjunction_maneuver_scratch_bytes(t: u32, bytes: *u64) i32;
pub extern fn astroz_cuda_correlate(elements: ?[*]const f64, n: u32, grav: i32, covariance: ?[*]const f64, model: ?[*]const u8, offsets: ?[*]const u32, t: u32, jd: ?[*]const f64, fr: ?[*]const f64, kind: ?[*]const u8, value: ?[*]const f64, sigma: ?[*]const f64, station: ?[*]const u32, m: u32, stations: ?[*]const f64, k: u32, gate_probability: f64, best: u32, device: i32, rows: ?[*]u32, d2: ?[*]f64, used: ?[*]u32, n_gate: ?[*]u32, n_failed: ?[*]u32, status: ?[*]u8, row_status: ?[*]u8) i32;
pub extern fn astroz_cuda_correlate_device(d_elements: ?[*]const f64, n: u32, grav: i32, d_covariance: ?[*]const f64, d_model: ?[*]const u8, d_offsets: ?[*]const u32, t: u32, d_jd: ?[*]const f64, d_fr: ?[*]const f64, d_kind: ?[*]const u8, d_value: ?[*]const f64, d_sigma: ?[*]const f64, d_station: ?[*]const u32, d_stations: ?[*]const f64, gate_probability: f64, best: u32, device: i32, d_scratch: ?*anyopaque, d_rows: ?[*]u32, d_d2: ?[*]f64, d_used: ?[*]u32, d_n_gate: ?[*]u32, d_n_failed: ?[*]u32, d_status: ?[*]u8, d_row_status: ?[*]u8, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_correlate_scratch_bytes(n: u32, t: u32, best: u32, bytes: *u64) i32;
pub extern fn astroz_cuda_chi2_quantile(k: u32, p: f64, x: ?[*]f64) i32;
pub extern fn astroz_cuda_tasking(elements: ?[*]const f64, n: u32, grav: i32, covariance: ?[*]const f64, model: ?[*]const u8, kind: ?[*]const u8, station: ?[*]const u32, sigma: ?[*]const f64, limits: ?[*]const f64, s: u32, stations: ?[*]const f64, k: u32, jd: ?[*]const f64, fr: ?[*]const f64, t: u32, sun: ?[*]const f64, gain_min: f64, device: i32, task_row: ?[*]u32, task_gain: ?[*]f64, task_value: ?[*]f64, task_spread: ?[*]f64, n_candidates: ?[*]u32, posterior: ?[*]f64, n_tasks: ?[*]u32, n_visible: ?[*]u32, n_failed: ?[*]u32, row_status: ?[*]u8) i32;
pub extern fn astroz_cuda_tasking_device(d_elements: ?[*]const f64, n: u32, grav: i32, d_covariance: ?[*]const f64, d_model: ?[*]const u8, d_kind: ?[*]const u8, d_station: ?[*]const u32, d_sigma: ?[*]const f64, d_limits: ?[*]const f64, s: u32, d_stations: ?[*]const f64, d_jd: ?[*]const f64, d_fr: ?[*]const f64, t: u32, d_sun: ?[*]const f64, gain_min: f64, device: i32, d_scratch: ?*anyopaque, d_task_row: ?[*]u32, d_task_gain: ?[*]f64, d_task_value: ?[*]f64, d_task_spread: ?[*]f64, d_n_candidates: ?[*]u32, d_posterior: ?[*]f64, d_n_tasks: ?[*]u32, d_n_visible: ?[*]u32, d_n_failed: ?[*]u32, d_row_status: ?[*]u8, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_tasking_scratch_bytes(n: u32, s: u32, bytes: *u64) i32;
pub extern fn astroz_cuda_initial_orbits(offsets: ?[*]const u32, t: u32, jd: ?[*]const f64, fr: ?[*]const f64, kind: ?[*]const u8, value: ?[*]const f64, sigma: ?[*]const f64, station: ?[*]const u32, m: u32, stations: ?[*]const f64, k: u32, bstar: ?[*]const f64, grav: i32, device: i32, elements: ?[*]f64, state: ?[*]f64, wrms: ?[*]f64, method: ?[*]u8, candidates: ?[*]u32, conv: ?[*]f64, deep_space: ?[*]u8, status: ?[*]u8) i32;
pub extern fn astroz_cuda_initial_orbits_device(d_offsets: ?[*]const u32, t: u32, d_jd: ?[*]const f64, d_fr: ?[*]const f64, d_kind: ?[*]const u8, d_value: ?[*]const f64, d_sigma: ?[*]const f64, d_station: ?[*]const u32, d_stations: ?[*]const f64, d_bstar: ?[*]const f64, grav: i32, device: i32, d_scratch: ?*anyopaque, d_elements: ?[*]f64, d_state: ?[*]f64, d_wrms: ?[*]f64, d_method: ?[*]u8, d_candidates: ?[*]u32, d_conv: ?[*]f64, d_deep_space: ?[*]u8, d_status: ?[*]u8, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_initial_orbits_scratch_bytes(t: u32, bytes: *u64) i32;
pub extern fn astroz_cuda_link_tracks(offsets: ?[*]const u32, t: u32, jd: ?[*]const f64, fr: ?[*]const f64, kind: ?[*]const u8, value: ?[*]const f64, sigma: ?[*]const f64, station: ?[*]const u32, m: u32, stations: ?[*]const f64, k: u32, pairs: ?[*]const u32, p: u32, bstar: ?[*]const f64, r_min: f64, r_max: f64, max_revs: u32, grav: i32, device: i32, elements: ?[*]f64, state: ?[*]f64, rho: ?[*]f64, revs: ?[*]u8, flags: ?[*]u8, wrms: ?[*]f64, used: ?[*]u32, hypotheses: ?[*]u32, conv: ?[*]f64, deep_space: ?[*]u8, status: ?[*]u8) i32;
pub extern fn astroz_cuda_link_tracks_device(d_offsets: ?[*]const u32, t: u32, d_jd: ?[*]const f64, d_fr: ?[*]const f64, d_kind: ?[*]const u8, d_value: ?[*]const f64, d_sigma: ?[*]const f64, d_station: ?[*]const u32, d_stations: ?[*]const f64, d_pairs: ?[*]const u32, p: u32, d_bstar: ?[*]const f64, r_min: f64, r_max: f64, max_revs: u32, grav: i32, device: i32, d_scratch: ?*anyopaque, d_elements: ?[*]f64, d_state: ?[*]f64, d_rho: ?[*]f64, d_revs: ?[*]u8, d_flags: ?[*]u8, d_wrms: ?[*]f64, d_used: ?[*]u32, d_hypotheses: ?[*]u32, d_conv: ?[*]f64, d_deep_space: ?[*]u8, d_status: ?[*]u8, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_link_tracks_scratch_bytes(p: u32, bytes: *u64) i32;
pub extern fn astroz_cuda_parse_tle(line1: [*:0]const u8, line2: [*:0]const u8, elements: ?[*]f64) i32;
pub extern fn astroz_cuda_lambert(r1: ?[*]const f64, r2: ?[*]const f64, tof: ?[*]const f64, normal: ?[*]const f64, n: u32, mu: f64, max_revs: u32, device: i32, v1: ?[*]f64, v2: ?[*]f64, status: ?[*]u8, iterations: ?[*]u8) i32;
pub extern fn astroz_cuda_lambert_device(d_r1: ?[*]const f64, d_r2: ?[*]const f64, d_tof: ?[*]const f64, d_normal: ?[*]const f64, n: u32, mu: f64, max_revs: u32, device: i32, d_v1: ?[*]f64, d_v2: ?[*]f64, d_status: ?[*]u8, d_iterations: ?[*]u8, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_lambert_porkchop_device(d_dep: ?[*]const f64, d_dep_status: ?[*]const u8, d_arr: ?[*]const f64, d_arr_status: ?[*]const u8, n_pairs: u32, d_dep_jd: ?[*]const f64, d_dep_fr: ?[*]const f64, n_dep: u32, d_arr_jd: ?[*]const f64, d_arr_fr: ?[*]const f64, n_arr: u32, mu: f64, max_revs: u32, device: i32, d_dv: ?[*]f64, d_slot: ?[*]u8, d_status: ?[*]u8, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_constellation_porkchop(h: Handle, chaser: ?[*]const u32, target: ?[*]const u32, n_pairs: u32, dep_jd: ?[*]const f64, dep_fr: ?[*]const f64, n_dep: u32, arr_jd: ?[*]const f64, arr_fr: ?[*]const f64, n_arr: u32, mu: f64, max_revs: u32, dv: ?[*]f64, slot: ?[*]u8, status: ?[*]u8) i32;
pub extern fn astroz_cuda_reentry(elements: ?[*]const f64, n: u32, grav: i32, covariance: ?[*]const f64, model: ?[*]const u8, rows: ?[*]const u32, ballistic: ?[*]const f64, samples: ?[*]const u64, first: ?[*]const u64, seed: ?[*]const u64, m: u32, h_i: f64, horizon_days: f64, step_s: f64, density_scale: f64, density_sigma: f64, record: u32, device: i32, record_out: ?[*]f64, states: ?[*]f64, nominal_status: ?[*]u8, counts: ?[*]u64, sample_out: ?[*]f64, status: ?[*]u8) i32;
pub extern fn astroz_cuda_reentry_device(d_elements: ?[*]const f64, n: u32, grav: i32, d_covariance: ?[*]const f64, d_model: ?[*]const u8, d_rows: ?[*]const u32, d_ballistic: ?[*]const f64, d_samples: ?[*]const u64, d_first: ?[*]const u64, d_seed: ?[*]const u64, m: u32, h_i: f64, horizon_days: f64, step_s: f64, density_scale: f64, density_sigma: f64, record: u32, device: i32, d_record_out: ?[*]f64, d_states: ?[*]f64, d_nominal_status: ?[*]u8, d_counts: ?[*]u64, d_sample_out: ?[*]f64, d_status: ?[*]u8, d_scratch: ?*anyopaque, stream: ?*anyopaque) i32;
pub extern fn astroz_cuda_reentry_scratch_bytes(m: u32, bytes: *u64) i32;
pub extern fn astroz_cuda_fp64_peak(device: i32, tflops: ?[*]f64) i32;
pub extern fn astroz_cuda_fp64_pipe_peak(device: i32, tflops: ?[*]f64) i32;

/// C API code -> the error set of the kernel-level boundary it replaces (src/simdKernels.zig:30-37)
pub fn toError(rc: i32) ?@import("../Sgp4.zig").Error {
    return switch (rc) {
        0 => null,
        -12 => error.SatelliteDecayed,
        -11 => error.InvalidEccentricity,
        -10 => error.DeepSpaceNotSupported,
        else => error.OutOfMemory, // -100 alloc, -200 CUDA, -201 no device: no CPU fallback is attempted
    };
}
