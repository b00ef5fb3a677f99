/*
 * pwpp.h — thin C-ABI of the H100 ground-segmentation engine (libpwpp_b200.so).
 *
 * This is the drop-in boundary for ONE path of url-kaist/patchwork-plusplus:
 * patchwork::PatchWorkpp::estimateGround() and the getters that read its result.
 * Everything above this header (the C++ class `patchwork::PatchWorkpp` in
 * include/patchwork/patchworkpp.h and the Python module `pypatchworkpp`) is glue.
 * No torch / Eigen / STL types cross this boundary: plain pointers, sizes, PODs.
 *
 * Each entry point cites the reference interface it replaces (paths relative to the
 * reference checkout, commit b608129a):
 *   H  = cpp/patchworkpp/include/patchwork/patchworkpp.h
 *   S  = cpp/patchworkpp/src/patchworkpp.cpp
 *   PB = python/patchworkpp/pybinding.cpp
 *
 * Model: a `pwpp_ctx` owns `num_streams` independent sensor streams. One stream is what
 * the reference calls one PatchWorkpp instance (H:114-235): it carries the temporal state
 * (adaptive elevation/flatness thresholds, their histories, the adaptive sensor height —
 * S:338-375) from frame to frame. pwpp_estimate_host / pwpp_estimate_device process ONE frame
 * for each of the first `nframes` streams, all on the GPU, in a single launch sequence. The
 * *_streams variants take a stream table instead: frame f of the call belongs to stream
 * streams[f], any subset of the streams in any order, a stream possibly several times (its
 * frames then run in call order, see "Stream table" below). The reference class maps to a ctx
 * with num_streams == 1.
 *
 * Indexing rule: everything a call PRODUCES is indexed by the frame's position f in the call
 * (counts, index lists, xyz, centers, normals, patch records, bin ids, pwpp_device_results,
 * pwpp_host_results); the temporal STATE is indexed by stream id (pwpp_get_state, pwpp_height,
 * pwpp_copy_history, pwpp_export_state / pwpp_import_state, pwpp_reset_stream). With the
 * identity table of pwpp_estimate_host / pwpp_estimate_device the two coincide. The PARAMETERS a frame
 * runs with are those of its stream's set (pwpp_create_sets; one set for a ctx from pwpp_create): results
 * by call position, state by stream id, parameters by the stream's set.
 *
 * All functions returning int return PWPP_OK (0) or a negative pwpp_status; the message
 * for the last failure on the calling thread is available from pwpp_last_error().
 * There is NO CPU fallback: creating a ctx without a usable CUDA device fails loudly.
 */
#ifndef PWPP_H_
#define PWPP_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PWPP_ABI_VERSION 1
#define PWPP_NUM_ZONES 4            /* H:127-134 hard-wires 4 zones via .at(0..3)          */
#define PWPP_MAX_RINGS_OF_INTEREST 4 /* H:174-175: update_flatness_[4], update_elevation_[4] */
#define PWPP_MAX_PARAM_SETS 8       /* parameter sets of one ctx (pwpp_create_sets) */

typedef enum pwpp_status {
  PWPP_OK = 0,
  PWPP_ERR_INVALID_ARG = -1,
  PWPP_ERR_CUDA = -2,
  PWPP_ERR_NO_DEVICE = -3,
  PWPP_ERR_UNSUPPORTED = -4,
  PWPP_ERR_CAPACITY = -5
} pwpp_status;

/* POD mirror of patchwork::Params (H:42-112); field names, meaning and defaults identical.
 * The std::vector fields become fixed [4] arrays (the reference only ever reads 4 entries).
 * `intensity_thr` is bound in Python (PB:37) but never read by the algorithm; kept for shape. */
typedef struct pwpp_params {
  int32_t verbose;                 /* H:44  (bool) */
  int32_t enable_RNR;              /* H:45  */
  int32_t enable_RVPF;             /* H:46  */
  int32_t enable_TGR;              /* H:47  */
  int32_t num_iter;                /* H:49  default 3  */
  int32_t num_lpr;                 /* H:50  default 20 */
  int32_t num_min_pts;             /* H:51  default 10 */
  int32_t num_zones;               /* H:52  must be 4  */
  int32_t num_rings_of_interest;   /* H:53  default 4, must be <= 4 */
  int32_t max_flatness_storage;    /* H:72  default 1000 */
  int32_t max_elevation_storage;   /* H:73  default 1000 */
  int32_t _pad0;
  double RNR_ver_angle_thr;        /* H:55  default -15.0 */
  double RNR_intensity_thr;        /* H:56  default 0.2   */
  double sensor_height;            /* H:58  default 1.723 (adaptive, S:348) */
  double th_seeds;                 /* H:59  default 0.125 */
  double th_dist;                  /* H:60  default 0.125 */
  double th_seeds_v;               /* H:61  default 0.25  */
  double th_dist_v;                /* H:62  default 0.1   */
  double max_range;                /* H:63  default 80.0  */
  double min_range;                /* H:64  default 2.7   */
  double uprightness_thr;          /* H:65  default 0.707 */
  double adaptive_seed_selection_margin; /* H:66 default -1.2 */
  double intensity_thr;            /* H:67  unused by the algorithm */
  int32_t num_sectors_each_zone[PWPP_NUM_ZONES]; /* H:69 default {16,32,54,32} */
  int32_t num_rings_each_zone[PWPP_NUM_ZONES];   /* H:70 default {2,4,4,4}     */
  double elevation_thr[PWPP_MAX_RINGS_OF_INTEREST]; /* H:75 default {0,0,0,0} (adaptive) */
  double flatness_thr[PWPP_MAX_RINGS_OF_INTEREST];  /* H:76 default {0,0,0,0} (adaptive) */
} pwpp_params;

/* Fills *p with the reference defaults (H:79-111). */
void pwpp_params_default(pwpp_params* p);

/* Temporal state of one stream — exactly the members the reference mutates between frames
 * (S:347-350, S:368, S:255-256, S:354-355, S:372-373). Used by tests and for
 * checkpoint / stream migration between GPUs. Histories hold at most
 * max_*_storage + (max bins per ring) entries; `hist_cap` is the row capacity in doubles.
 * BOUND (defined deviation, DESIGN.md section 3): a history row keeps its newest
 * hist_cap = max(max_elevation_storage, max_flatness_storage) + 4 * (max sectors of a zone) + 64 samples. The reference's
 * vectors are unbounded while ring 0 holds <= 1 flatness samples (the `break` of S:363-364 then skips the trimming of rings
 * 1..3); after more than hist_cap accepted patches of one ring in that state the reference averages over the whole history, this
 * library over the newest hist_cap samples. The state blob of pwpp_export_state depends on hist_cap (checked on import).
 * NO-PLANE PATCHES (defined deviation): a patch all of whose seed sets are empty has no plane of its own; the reference
 * (S:49) then partitions it with the normal_/d_ left behind by the previous estimate_plane call. Here all points of such a patch
 * are non-ground and A-GLE sees the carried mean / normal / singular values (pwpp_bin_result.verdict == -1 marks the patch). */
typedef struct pwpp_state {
  double sensor_height;
  double elevation_thr[PWPP_MAX_RINGS_OF_INTEREST];
  double flatness_thr[PWPP_MAX_RINGS_OF_INTEREST];
  int32_t n_elevation[PWPP_MAX_RINGS_OF_INTEREST];
  int32_t n_flatness[PWPP_MAX_RINGS_OF_INTEREST];
} pwpp_state;

typedef struct pwpp_ctx pwpp_ctx;

/* ---- lifetime -------------------------------------------------------------------------- */

/* Replaces PatchWorkpp::PatchWorkpp(Params) (H:120-150): builds the concentric-zone geometry
 * (H:122-134) and `num_streams` fresh stream states on CUDA device `device`.
 * `max_points_per_frame` sizes the per-frame device buffers (frames may be smaller);
 * capacity grows on demand if a later call exceeds it. */
int pwpp_create(const pwpp_params* params, int device, int num_streams,
                int64_t max_points_per_frame, pwpp_ctx** out);

/* Several parameter sets in one ctx: stream s runs with sets[stream_set[s]] for its whole life, exactly like a
 * reference instance constructed with those Params (H:120), and one call may mix streams of any sets. Per-frame
 * results follow the frame's set: pwpp_copy_bin_results writes that set's nbins records, pwpp_copy_bin_ids uses its
 * pseudo-bin ids (nbins, nbins + 1), centers / normals / patch counts cover its bins. State follows the stream's set:
 * reset restores the set's sensor_height / elevation_thr / flatness_thr, the history bound (hist_cap, see pwpp_state)
 * is the set's own, and a stream's state blob is the one a one-set ctx with that set produces (importable either way).
 * Every set goes through the checks of pwpp_create; num_sets must be in [1, PWPP_MAX_PARAM_SETS] and stream_set a
 * non-NULL array of num_streams ids in [0, num_sets). A failure returns PWPP_ERR_INVALID_ARG or PWPP_ERR_UNSUPPORTED
 * (the message names the set) before anything is allocated. pwpp_create is this with one set. */
int pwpp_create_sets(const pwpp_params* sets, int num_sets, const int32_t* stream_set, int device, int num_streams,
                     int64_t max_points_per_frame, pwpp_ctx** out);
void pwpp_destroy(pwpp_ctx* ctx);

const char* pwpp_last_error(void);
int pwpp_abi_version(void);
/* Number of polar bins of the configured concentric-zone model (504 with defaults). With several parameter sets: the
 * largest bin count of the sets (a pwpp_copy_bin_results buffer of that size fits any frame). */
int pwpp_num_bins(const pwpp_ctx* ctx);
/* Bin count of stream s's parameter set, and the set id of stream s (negative status for a bad s). */
int pwpp_stream_num_bins(const pwpp_ctx* ctx, int s);
int pwpp_stream_set(const pwpp_ctx* ctx, int s);

/* ---- the hot path ---------------------------------------------------------------------- */

/* Replaces PatchWorkpp::estimateGround(Eigen::MatrixXf) (H:152, S:151-336) for HOST buffers.
 * Frame f (0 <= f < nframes <= num_streams) is read from pts[f]: n[f] points of `cols`
 * (3 or 4) floats; element (i,c) is at pts[f][i*row_stride + c*col_stride] (so both numpy
 * C-order N x C and Eigen column-major N x C are accepted without a caller-side copy).
 * cols == 3 disables RNR for that call exactly like S:379-382.
 * Copies host->device through pinned staging, runs all stages on the GPU, and leaves the
 * results on the device; the copy_* getters below fetch them. The caller's buffers are
 * never modified (the reference mutates only its by-value copy, S:394). */
int pwpp_estimate_host(pwpp_ctx* ctx, int nframes, const float* const* pts, const int64_t* n,
                       int cols, int64_t row_stride, int64_t col_stride);

/* Same path for DEVICE-resident input (used by the benchmark's device-resident leg and by
 * GPU pipelines): `d_pts` is a device pointer to packed float4 {x,y,z,intensity} points of
 * all frames back to back; frame f occupies [h_offsets[f], h_offsets[f+1]) (host array of
 * nframes+1 int64). `has_intensity` == 0 behaves like cols == 3. `cuda_stream` is a
 * cudaStream_t (may be NULL = the ctx's own stream). Asynchronous w.r.t. the host: results
 * are ready after pwpp_synchronize() (the copy_* getters synchronize themselves). */
int pwpp_estimate_device(pwpp_ctx* ctx, int nframes, const void* d_pts,
                         const int64_t* h_offsets, int has_intensity, void* cuda_stream);

/* The same for packed N x 3 rows {x, y, z} resident on the device (no intensity: RNR is skipped like for N x 3 host input,
 * S:379-382): the rows are padded to the kernels' 16-byte points by a device-side copy into the ctx's input buffer. */
int pwpp_estimate_device_xyz(pwpp_ctx* ctx, int nframes, const void* d_xyz, const int64_t* h_offsets, void* cuda_stream);

/* Stream table: the same two paths with frame f of the call belonging to stream streams[f]
 * (0 <= streams[f] < num_streams; 1 <= nframes <= 65535, nframes may exceed num_streams).
 *   - Any subset of the streams, in any order. Streams the call does not name keep their state untouched.
 *   - A stream may appear several times: its frames are processed in call order, each one sees the state the
 *     previous one left (exactly as in separate calls). The call is split into maximal runs of consecutive
 *     frames with pairwise distinct streams; each run is one launch sequence over its frames, and stream
 *     order serialises the runs. In pwpp_estimate_host the launch ranges are its pipeline chunks cut at the
 *     run boundaries, so the upload of later frames still overlaps the kernels of earlier ones.
 *   - Results are indexed by call position f, state by stream id (the indexing rule above).
 *   - A NULL table, an id out of range or nframes outside [1, 65535] returns PWPP_ERR_INVALID_ARG before anything
 *     is launched: no stream's state changes.
 * pwpp_estimate_host / pwpp_estimate_device are these with the identity table streams[f] = f. */
int pwpp_estimate_host_streams(pwpp_ctx* ctx, int nframes, const int32_t* streams, const float* const* pts, const int64_t* n,
                               int cols, int64_t row_stride, int64_t col_stride);
int pwpp_estimate_device_streams(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* d_pts, const int64_t* h_offsets,
                                 int has_intensity, void* cuda_stream);

/* ---- sensor point records of any PointCloud2 layout ------------------------------------------------------------------
 * A frame may also be handed over as the sensor driver published it: n[f] records of layouts[f].point_step bytes starting at
 * frames[f] (any alignment, any step: 22, 13 and 17 are as valid as 16), with the byte offset and datatype of the x, y, z and
 * intensity fields inside a record (sensor_msgs/PointField). One kernel unpacks every frame of a launch range on the GPU into
 * the ctx's own float4 input buffer; everything after that is the path of pwpp_estimate_host / pwpp_estimate_device.
 *   - Every frame carries its own layout, so one call may mix sensors of different drivers. Results by call position, state
 *     by stream id, parameters by the stream's set, layout by the frame. The stream table (required, non-NULL) works exactly
 *     as for the *_streams entry points: same checks, same error codes, same run splitting.
 *   - Fields are converted to float by value with round-to-nearest-even (numpy's astype(np.float32)); FLOAT32 passes through
 *     bit for bit. A FLOAT64 NaN becomes the quiet float NaN with the same sign and the top payload bits. Records are
 *     little-endian.
 *   - A frame whose layout has no intensity field (offset[3] < 0) is segmented exactly like an N x 3 frame (RNR skipped,
 *     S:379-382), even when other frames of the call carry intensity: its points get a NaN intensity, which no RNR test
 *     accepts, and the call runs with intensity on when any of its frames has it.
 *   - No byte outside [frames[f], frames[f] + n[f] * point_step) is read.
 *   - Checked before anything is allocated or launched (the message names the frame and the field); no stream's state
 *     changes on an error. PWPP_ERR_INVALID_ARG: a NULL streams / frames / n / layouts array, a NULL frame pointer with
 *     n > 0, n < 0, point_step < 1, an unknown datatype code, a field that does not fit inside point_step.
 *     PWPP_ERR_UNSUPPORTED: x / y / z not FLOAT32 or FLOAT64, point_step > PWPP_MAX_POINT_STEP.
 *   - After the call the unpacked points live in the ctx: every getter works as after the other entry points, and the xyz
 *     getters stay correct after the caller frees or reuses its record buffer.
 * pwpp_launch_count rises by one unpack launch per pipeline chunk that holds points (host) or per call (device). */
#define PWPP_FIELD_INT8 1    /* sensor_msgs/PointField datatype codes */
#define PWPP_FIELD_UINT8 2
#define PWPP_FIELD_INT16 3
#define PWPP_FIELD_UINT16 4
#define PWPP_FIELD_INT32 5
#define PWPP_FIELD_UINT32 6
#define PWPP_FIELD_FLOAT32 7
#define PWPP_FIELD_FLOAT64 8
#define PWPP_MAX_POINT_STEP 1024

typedef struct pwpp_point_layout {
  int32_t point_step;   /* bytes from one point to the next (PointCloud2::point_step), 1..PWPP_MAX_POINT_STEP */
  int32_t offset[4];    /* byte offsets of x, y, z, intensity inside a point; offset[3] < 0: no intensity field */
  int32_t datatype[4];  /* PWPP_FIELD_*; x, y, z must be FLOAT32 or FLOAT64, intensity any of the eight */
} pwpp_point_layout;

/* Host-resident records. Every frame's bytes travel as they are (no per-point host loop): a page-locked buffer by DMA
 * straight from it, a pageable one by one memcpy into page-locked staging and then DMA. The unpack runs on the upload stream
 * of the pipeline, so pwpp_call_times_us's host->device phase includes it. */
int pwpp_estimate_host_records(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* const* frames,
                               const int64_t* n, const pwpp_point_layout* layouts /* [nframes] */);
/* Device-resident records: unpacked on `cuda_stream` (NULL = the ctx's own stream) with the stream-ordering rules of
 * pwpp_estimate_device_xyz; the records must stay untouched until the call's work on that stream has run, and, when the
 * record results below are wanted, until they have been fetched (their gather reads the caller's buffers). */
int pwpp_estimate_device_records(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* const* d_frames,
                                 const int64_t* n, const pwpp_point_layout* layouts /* [nframes] */, void* cuda_stream);

/* Results of the last RECORDS call (pwpp_estimate_*_records) as records of each frame's own layout: every field the sensor
 * sent (intensity, ring, per-point time, padding) comes back byte for byte, so a ROS 2 node can publish its ground and
 * non-ground clouds with the input's fields. Frame f's region starts at byte h_offsets[f] (16-byte aligned; h_offsets has
 * nframes + 1 entries): num_ground(f) ground records, then num_nonground(f) non-ground records, in index-list order (record k
 * is input record k of the frame's lists, PWPP_ORDER_BIN or PWPP_ORDER_REFERENCE as the call ran); the bytes after them in
 * the region are unspecified.
 *   - The first of these four functions called after a call gathers the records of every frame in one kernel on the GPU
 *     (pwpp_launch_count rises by one; none for a call without points), on the call's stream; later calls of them reuse it.
 *     The host view adds one device->host copy into a page-locked buffer, and the per-frame getters copy from that. Calls
 *     that never ask for record results allocate and launch nothing for them.
 *   - Host blocking of pwpp_device_record_results: none once its buffers are warm, i.e. after a request of a call at least as
 *     large (in frames and record bytes). A request that first reserves or grows the output buffers or their page-locked
 *     offset table allocates device / page-locked memory, which the CUDA runtime may synchronize; and a request waits for the
 *     previous request's offset-table upload to have run (enqueued one call earlier, so in practice long done).
 *   - PWPP_ERR_INVALID_ARG before any call, for a frame outside the last call, and when the last call did not take records
 *     (the xyz getters serve those). Valid until the next estimate call. */
int pwpp_device_record_results(pwpp_ctx* ctx, const void** d_records, const int64_t** h_offsets);  /* enqueued on the call's stream; no host sync once warm */
int pwpp_host_record_results(pwpp_ctx* ctx, const void** h_records, const int64_t** h_offsets);    /* page-locked view, one D2H */
int pwpp_copy_ground_records(pwpp_ctx* ctx, int f, void* dst);       /* num_ground(f) * point_step bytes */
int pwpp_copy_nonground_records(pwpp_ctx* ctx, int f, void* dst);    /* num_nonground(f) * point_step bytes */

/* ---- bound calls: frame sizes read on the GPU, capturable into the caller's CUDA graph --------------------------------------
 * A GPU pipeline often knows a frame's size only on the device (a compaction kernel wrote it, or a static-shape pipeline pads
 * every frame to a capacity and carries the count as a device tensor). A BOUND call holds its frames, their capacities, the
 * device array of their counts and the stream table, fixed once by pwpp_bind_call. A ctx holds up to PWPP_MAX_BOUND_CALLS of
 * them; every entry point below acts on the selected one (pwpp_select_bound_call, "Several bound calls"). Running it needs only a
 * CUDA stream, performs no host synchronisation, and may be captured into the caller's CUDA graph; every run or replay reads
 * the current counts and frame contents.
 *
 * pwpp_bind_call: frame f is up to max_n[f] records of layouts[f] at device address frames[f] (any alignment, as in
 * pwpp_estimate_device_records), of stream streams[f]. Its size is d_counts[f] (device int64[nframes]), read by the GPU when
 * the call runs. Does all host work now: the checks of the records entry points (with n = max_n: the message names the
 * frame), the stream-table checks and the run split, and reserving every work buffer for sum(max_n) points. It uploads the
 * stream, set and record tables into buffers the bound call owns, then synchronizes. Binding ends the previous call's results
 * (the buffers they live in may move). PWPP_ERR_INVALID_ARG also when a call is already bound or d_counts is NULL.
 *
 * pwpp_run_bound_call: enqueues the bound call on cuda_stream (NULL = the ctx's own stream). Only kernels, device-to-device
 * work and event record / wait between the ctx's streams: no host synchronisation, no allocation and no host-memory copy. It
 * may be captured into a CUDA graph (global capture mode included); replays then read the current counts and frames. The
 * run makes the bound call the ctx's last call.
 *
 * pwpp_bound_call_results: device views of the bound call's results, at fixed addresses while it stays bound, laid out like
 * pwpp_device_results with the offsets on the device: *d_offsets int64[nframes + 1] (the exclusive scan of the accepted
 * counts: frame f's region of *d_indices starts there), *d_num_ground int32[nframes], *d_status int32[nframes]. Calling it
 * also makes the bound call the ctx's last call, so the per-frame host getters (pwpp_num_ground, pwpp_copy_*_indices,
 * centers, normals, bin results and ids, pwpp_host_results) serve its results after a run or a graph replay; they fetch the
 * offsets with their first device->host copy. After a replay the caller synchronizes with the replay's stream before using
 * the host getters (they only synchronize with the stream of the last pwpp_run_bound_call).
 *
 * Rules:
 *   - Out-of-range counts. A count outside [0, max_n[f]] cannot return an error from a replay: frame f runs as an empty
 *     frame instead, exactly as a direct call with n = 0 would, its stream state advances as after that empty call, and
 *     d_status[f] = PWPP_COUNT_OUT_OF_RANGE (0 otherwise). The other frames are unaffected. Nothing past
 *     frames[f] + max_n[f] * point_step is ever read.
 *   - Buffers are frozen while a call is bound, so no buffer a captured graph holds ever moves:
 *       a direct call that would grow a work buffer returns PWPP_ERR_CAPACITY before anything runs, and no state changes
 *       (a direct call that fits runs as usual);
 *       pwpp_set_output_order returns PWPP_ERR_INVALID_ARG: the bound call keeps the order it was bound with.
 *     pwpp_unbind_call lifts the freeze and makes graphs that hold the bound call invalid.
 *   - Shared state and results. Direct calls and runs of the bound call use the same stream state and the same result
 *     buffers; each one's results are valid until the next call or replay. The caller orders replays against direct calls
 *     (same stream, or its own events): the ctx cannot see a replay, and a capture cannot wait on an event recorded outside it.
 *   - pwpp_launch_count rises, per pwpp_run_bound_call, by one table launch, one unpack launch when any max_n > 0, the
 *     usual launch sequence of each run (grids sized for the capacities), and, once record results are enabled
 *     (pwpp_bind_record_results), one gather launch, also when every max_n is 0.
 *   - The record results of direct calls (pwpp_*_record_results, pwpp_copy_*_records) refuse a bound call with a message:
 *     their gather needs host offsets. A bound call has record results of its own (below).
 *
 * Record results of the bound call: its ground and non-ground clouds as records of each frame's own layout (every field the
 * sensor sent, byte for byte), gathered on the GPU at fixed addresses, for consumers that slice them without knowing any count
 * on the host (a CUDA graph, a static-shape torch pipeline, a publisher of device buffers).
 *
 * pwpp_bind_record_results: enables them for the bound call. parts is PWPP_PART_GROUND, PWPP_PART_NONGROUND or both (3). Host
 * work like pwpp_bind_call (it reserves the buffers, then synchronizes), so it is not capturable; graphs captured before it do
 * not gather. From then on every pwpp_run_bound_call ends with one gather launch on its stream, after the last run's output
 * kernel, with no host work. PWPP_ERR_INVALID_ARG when no call is bound, for parts outside {1, 2, 3}, and when record results
 * are already enabled (one setting per bind: pwpp_unbind_call releases them, and a later bind starts with them off).
 *
 * Layout: one device buffer per enabled part. Frame f owns bytes [off[f], off[f + 1]) of each, off[f + 1] = off[f] +
 * align16(max_n[f] * point_step_f) (the direct call's offsets with n = max_n; the same for both buffers). Every run writes, for
 * every frame, num_ground(f) records at the start of the frame's ground region and num_nonground(f) records at the start of its
 * non-ground region, record k = input record k of that list in the order the call was bound with (PWPP_ORDER_BIN or
 * PWPP_ORDER_REFERENCE), and d_counts[2f] = ground, d_counts[2f + 1] = non-ground (int32), both counts whichever parts are
 * enabled. A frame whose count was out of range ran as empty: its counts are 0 and its regions are not written. Bytes of a
 * region past its count are never written. Memory: sum over frames of align16(max_n[f] * point_step_f) bytes per enabled part,
 * plus 8 (nframes + 1) + 8 nframes bytes. The buffers are not work buffers: reserving them does not interact with the freeze.
 *
 * pwpp_bound_record_results: host-only. The fixed device pointers of the two buffers (NULL for a part that is not enabled), the
 * host offsets off (nframes + 1) and the device counts int32[2 nframes]. PWPP_ERR_INVALID_ARG when no call is bound or record
 * results are not enabled. Direct records calls between runs keep their own record results and never touch these buffers. */
#define PWPP_COUNT_OUT_OF_RANGE 1   /* d_status[f]: d_counts[f] < 0 or > max_n[f]; the frame was run as an empty frame */
int pwpp_bind_call(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* const* frames, const int64_t* max_n,
                   const pwpp_point_layout* layouts, const int64_t* d_counts);

/* Per-frame actions of a bound call, for sensors that do not tick together: a frame can be left out of a run, or its stream
 * reset first, decided on the GPU at every run or replay. A count of 0 is not the same as leaving a frame out: an empty frame
 * still runs the threshold update, which moves the state of a stream whose histories are full.
 *
 * pwpp_bind_call_actions: pwpp_bind_call plus d_actions, a device int32 array of nframes actions that the GPU reads at every
 * run or replay, like d_counts. d_actions == NULL is exactly pwpp_bind_call. The actions are a bind argument because skipping
 * needs scratch state slots (below), and reserving them later would move the state buffers under a graph already captured.
 *   - PWPP_FRAME_RUN: the frame runs as with pwpp_bind_call.
 *   - PWPP_FRAME_SKIP: the frame is absent from this run. It runs as an empty frame whose count is neither read nor
 *     validated; its stream's complete state (the export blob: histories and the carried plane included) stays bit for bit
 *     what it was. Its results by position are those of an empty frame (an empty list span in the offsets, num_ground 0, no
 *     patches), its record-result counts are 0 and its record regions are not written. d_status[f] = PWPP_FRAME_SKIPPED.
 *   - PWPP_FRAME_RESET: the stream is restored to its set's constructor state, as by pwpp_reset_stream, immediately before
 *     this frame (after the stream's earlier frames of the bound call have run), then the frame runs as RUN would. An
 *     out-of-range count still gives PWPP_COUNT_OUT_OF_RANGE and an empty frame, with the reset applied; RESET with count 0
 *     is "reset only": the state equals a freshly reset stream's, bit for bit.
 *   - Any other value: the frame is skipped and d_status[f] = PWPP_ACTION_INVALID (a replay cannot return an error).
 *   - Each run reads every action once, in its first kernel, into a copy the ctx owns; the later kernels of the run read the
 *     copy, so rewriting d_actions during a run never splits one frame's action between kernels.
 *   - pwpp_launch_count rises, compared with the same call bound without actions, by one reset launch for each run that holds
 *     a frame whose stream also has a frame in an earlier run. A bound call without repeated streams has no extra launch.
 *   - Scratch slots: a skipped frame is redirected to a scratch state slot, so the kernels see an ordinary empty frame and the
 *     real stream is never written. The bind grows the state and history buffers by L slots, L the longest run of the call (at
 *     most num_streams), sizeof(state) + 64 * history capacity bytes each (about 82 KB with the default parameters); the
 *     streams' states are copied across, a failed allocation leaves them as they were, and growing them makes graphs captured
 *     earlier by the ctx's own small calls capture again. The slots stay reserved after pwpp_unbind_call.
 *   - The freeze, pwpp_unbind_call and the record results behave as for pwpp_bind_call. */
#define PWPP_FRAME_RUN 0        /* the frame runs as with pwpp_bind_call */
#define PWPP_FRAME_SKIP 1       /* the frame is absent from this run */
#define PWPP_FRAME_RESET 2      /* reset the stream to its set's constructor state, then run the frame */
#define PWPP_FRAME_SKIPPED 2    /* d_status[f]: the frame's action was PWPP_FRAME_SKIP */
#define PWPP_ACTION_INVALID 3   /* d_status[f]: the frame's action was not a PWPP_FRAME_* value; it was skipped */
int pwpp_bind_call_actions(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* const* frames, const int64_t* max_n,
                           const pwpp_point_layout* layouts, const int64_t* d_counts, const int32_t* d_actions);

/* Scan rings of a bound call: a driver, a packet decoder or a DMA engine writes scan t + 1 into the next slot of a ring while
 * scan t is consumed. With rings the address of every frame is picked on the GPU at every run or replay, so the bound call
 * segments each scan in the slot where it was written, with no copy into a fixed buffer.
 *
 * pwpp_scan_ring: slot s of a ring holds d_counts[s] records starting at base + s * slot_stride (device memory, any alignment).
 *
 * pwpp_bind_call_rings: pwpp_bind_call_actions with the frames in rings. Frame f reads ring rings[f] (descriptors are copied at
 * bind time) and d_slots[f], a device int32 array of nframes slot numbers that the GPU reads at every run or replay, like the
 * counts. d_actions as for pwpp_bind_call_actions (NULL: all RUN).
 *   - Reading the slot. On every run or replay, frame f reads s = d_slots[f] once, in the run's first kernel, into a copy the ctx
 *     owns (pwpp_bound_call_slots). It then reads rings[f].d_counts[s] and segments the records at base + s * slot_stride.
 *     Everything else is as for pwpp_bind_call_actions: the count rule (a count outside [0, max_n[f]] gives
 *     PWPP_COUNT_OUT_OF_RANGE and an empty frame), the actions, the record results, the freeze and pwpp_unbind_call.
 *   - Precedence. A frame whose action skips it reads neither its slot nor a count (status PWPP_FRAME_SKIPPED or
 *     PWPP_ACTION_INVALID, slot copy -1). Otherwise a slot outside [0, num_slots) gives PWPP_SLOT_OUT_OF_RANGE: the frame runs as
 *     an empty frame and its stream advances as after an empty call, like an out-of-range count; a RESET still applies.
 *     Otherwise the count rule applies.
 *   - What is read. No byte outside [base, base + (num_slots - 1) * slot_stride + max_n[f] * point_step) is read, whatever
 *     d_slots holds.
 *   - Shared rings. Several frame entries may name the same ring, with identical descriptors: for example one sensor's backlog,
 *     its stream bound twice, the second entry reading the next slot or skipped.
 *   - The caller's obligation. Between a run's first kernel and the end of its last kernel (the record gather or the packed
 *     records gather, when enabled), the caller must not write a slot the run reads (its records or its count). Writing other slots, d_slots and other slots'
 *     counts is allowed and does not affect the run.
 *   - Bind-time checks, before anything is allocated, each message naming the frame (PWPP_ERR_INVALID_ARG): every check of
 *     pwpp_bind_call with frames[f] = base and n = max_n; NULL rings, d_slots or d_counts; NULL base with max_n > 0;
 *     num_slots < 1; slot_stride < max_n * point_step; a ring extent that overflows.
 *   - pwpp_launch_count rises exactly as for the same call bound with pwpp_bind_call_actions: there is no extra launch.
 *   - Identity. pwpp_bind_call_actions(frames, max_n, layouts, d_counts, d_actions) is this call with one-slot rings
 *     {frames[f], max_n[f] * point_step, d_counts + f, 1} and d_slots all zero, bit for bit.
 *   - Memory: 24 + 48 + 4 bytes per frame on the device, next to the bound call's other tables.
 *
 * pwpp_bound_call_slots: host-only. The ctx's copy of the slots the last run read, device int32[nframes] at a fixed address
 * while the call stays bound: the slot each frame read (also an out-of-range one), -1 where the action skipped the frame; -1
 * everywhere before the first run. PWPP_ERR_INVALID_ARG when no call is bound or it was bound without rings. */
typedef struct pwpp_scan_ring {
  const void* base;          /* device address of slot 0's first record (any alignment) */
  int64_t slot_stride;       /* bytes from slot s to slot s + 1; >= max_n[f] * point_step of every frame bound to it */
  const int64_t* d_counts;   /* device int64[num_slots]: the number of records in each slot, read by the GPU */
  int32_t num_slots;         /* >= 1 */
  int32_t _pad;
} pwpp_scan_ring;
#define PWPP_SLOT_OUT_OF_RANGE 4   /* d_status[f]: d_slots[f] < 0 or >= num_slots; the frame ran as an empty frame */
int pwpp_bind_call_rings(pwpp_ctx* ctx, int nframes, const int32_t* streams, const pwpp_scan_ring* rings /* [nframes] */,
                         const int64_t* max_n, const pwpp_point_layout* layouts, const int32_t* d_slots /* device [nframes] */,
                         const int32_t* d_actions /* NULL: all RUN */);
int pwpp_bound_call_slots(pwpp_ctx* ctx, const int32_t** d_slots_read);

/* Packed batches of a bound call: all frames back to back in one buffer, frame f at records [d_offsets[f], d_offsets[f + 1]),
 * the layout of torch.nested's jagged tensors, of PyG's ptr and of any stream compaction over a whole batch. The offsets live
 * on the device and may change at every tick, so where every frame starts is decided on the GPU at every run or replay, with
 * no scatter into fixed per-frame buffers.
 *
 * pwpp_bind_call_packed: pwpp_bind_call_actions with the frames in one packed buffer. base holds capacity records of *layout
 * (one point_step for the whole buffer, any alignment). d_offsets is a device int64 array of nframes + 1 entries that the GPU
 * reads at every run or replay; max_n[f] keeps its meaning (it bounds frame f's count and sizes the grids). d_actions as for
 * pwpp_bind_call_actions (NULL: all RUN).
 *   - Reading the offsets. On every run or replay, frame f reads lo = d_offsets[f] and hi = d_offsets[f + 1] in the run's first
 *     kernel. If lo < 0, hi < lo or hi > capacity, d_status[f] = PWPP_OFFSETS_OUT_OF_RANGE: the frame runs as an empty frame and
 *     its stream advances as after an empty call. Otherwise a count hi - lo above max_n[f] gives PWPP_COUNT_OUT_OF_RANGE and an
 *     empty frame. Otherwise the frame is the hi - lo records at base + lo * point_step. Each frame is judged by its own two
 *     entries only.
 *   - Precedence. A frame whose action skips it reads neither offset (status PWPP_FRAME_SKIPPED or PWPP_ACTION_INVALID). A
 *     RESET still applies when the frame's offsets turn out invalid.
 *   - What is read. No byte outside [base, base + capacity * point_step) is read, whatever d_offsets holds.
 *   - Results. Everything else is as for pwpp_bind_call_actions: the stream table and run split, the record results, the getter
 *     results, the freeze and pwpp_unbind_call. The index lists stay frame-relative (index k of frame f is record lo + k).
 *   - The caller's obligation. Between a run's first kernel and the end of its last kernel (the packed records gather, when
 *     enabled), the caller must not write the offsets or the records of the frames the run reads.
 *   - Bind-time checks, before anything is allocated, each message naming the frame or the field (PWPP_ERR_INVALID_ARG or
 *     PWPP_ERR_UNSUPPORTED): every check of pwpp_bind_call with frames[f] = base, layouts[f] = *layout and n = max_n[f]; NULL
 *     layout or d_offsets; NULL base with capacity > 0; capacity < 0; capacity * point_step or its end address overflowing.
 *   - Work buffers are reserved for sum(max_n) points, as for pwpp_bind_call. Accepted frames may overlap in the buffer (a
 *     decreasing offset makes its frame invalid, and a skipped frame validates neither of its entries, so the frames around it
 *     can share records), so the accepted counts of one run are bounded by sum(max_n), not by capacity.
 *   - pwpp_launch_count rises exactly as for the same call bound with pwpp_bind_call_actions: there is no extra launch.
 *   - Identity. With frames[f] = base + d_offsets[f] * point_step and d_counts[f] = d_offsets[f + 1] - d_offsets[f] (valid
 *     offsets), pwpp_bind_call_actions gives the same results bit for bit: indices, offsets, status, patches, states, record and
 *     getter results.
 *   - Memory: 48 + 48 bytes per frame on the device, next to the bound call's other tables.
 *
 * Packed xyz results of a bound call, for a consumer that takes one packed tensor with offsets rather than the capacity layout of
 * pwpp_bound_getters.
 *
 * pwpp_bind_packed_xyz: enables them for any bound call (plain, with actions, rings or packed). parts is PWPP_PART_GROUND,
 * PWPP_PART_NONGROUND or both (3). Host work that synchronizes, like pwpp_bind_getter_results, so it is not capturable; graphs
 * captured before it do not write these results. PWPP_ERR_INVALID_ARG when no call is bound, for parts outside {1, 2, 3}, and
 * when packed xyz is already enabled (one setting per bind: pwpp_unbind_call releases the buffers).
 *   - Layout. Per enabled part, a float32 buffer of rows of 3 and a device int64[nframes + 1] offsets array, the exclusive scan of
 *     that part's per-frame counts in the run. After every run or replay frame f's ground rows are ground[g_off[f] : g_off[f+1]]
 *     and its non-ground rows nonground[ng_off[f] : ng_off[f + 1]]. Row k of a frame is row k of pwpp_copy_ground_xyz /
 *     pwpp_copy_nonground_xyz of that frame, bit for bit, in the order the call was bound with. Skipped frames and frames with an
 *     invalid count, slot or offsets have count 0. Rows past off[nframes] are never written.
 *   - Independent of the getter results: both can be enabled, and each writes its own buffers.
 *   - pwpp_launch_count rises, per pwpp_run_bound_call, by two launches after the last run's output kernel (the offset scan and
 *     the gather), also when every max_n is 0. The offset scan is shared with packed records (below).
 *   - Memory: 12 sum(max_n) bytes per enabled part plus 16 (nframes + 1) bytes of offsets.
 *
 * pwpp_bound_packed_xyz: host-only. The fixed device pointers of both buffers and both offsets arrays (NULL for a part that is
 * not enabled). PWPP_ERR_INVALID_ARG when no call is bound or packed xyz is not enabled.
 *
 * Packed records of a bound call: the ground and non-ground clouds in the sensor's own record layout (every field, byte for
 * byte, as pwpp_bind_record_results writes them) with all frames back to back and device offsets, for a consumer that takes one
 * packed batch: a detector's (N, 4) xyzi batch with its batch offsets, a multi-sweep stage that needs each point's time, one
 * merged cloud published in the drivers' own layout.
 *
 * pwpp_bind_packed_records: enables them for any bound call (plain, with actions, rings or packed). parts is PWPP_PART_GROUND,
 * PWPP_PART_NONGROUND or both (3). Host work that synchronizes, so it is not capturable; graphs captured before it do not write
 * these results. PWPP_ERR_INVALID_ARG when no call is bound, for parts outside {1, 2, 3}, and when packed records are already
 * enabled (one setting per bind: pwpp_unbind_call releases the buffers). Every frame of the bound call must have the same
 * point_step, so that a part is one (rows, point_step) byte array (field offsets and datatypes may differ: the bytes are copied
 * as they are); otherwise PWPP_ERR_UNSUPPORTED, the message naming the first frame whose point_step differs from frame 0's.
 * Such a call keeps the capacity layout of pwpp_bind_record_results. The buffers are not work buffers: the freeze does not apply.
 *   - Layout. Per enabled part, one buffer of sum(max_n) records of point_step bytes and a device int64[nframes + 1] offsets array
 *     in records. After every run or replay frame f's records of a part are records [off[f], off[f + 1]) of that part's buffer,
 *     at byte off[f] * point_step, with no padding: neighbouring frames may share a 16-byte word. Record k of a frame is record k
 *     of its list in the order the call was bound with, byte for byte what pwpp_bind_record_results writes for the frame after
 *     the same run. Skipped frames and frames with an invalid count, slot or offsets have count 0. No byte at or past
 *     off[nframes] * point_step is written.
 *   - The offsets are packed xyz's: when both are enabled, pwpp_bound_packed_xyz and pwpp_bound_packed_records return the same
 *     two arrays, filled by one scan per run. The scan writes both arrays whichever parts are enabled.
 *   - pwpp_launch_count rises, per pwpp_run_bound_call, after the last run's output kernel, by one offset scan when packed xyz
 *     or packed records is enabled (one, not two, when both are) plus one gather per enabled feature, also when every max_n is 0.
 *   - The caller's obligation. The gather reads the caller's records, as the record results' gather does: the records a run
 *     reads stay unwritten until the end of this gather.
 *   - Direct calls between runs never write these buffers.
 *   - Memory: point_step sum(max_n) bytes per enabled part, plus 16 (nframes + 1) bytes of offsets unless packed xyz is enabled.
 *
 * pwpp_bound_packed_records: host-only. The fixed device pointers of both buffers and both offsets arrays (NULL for a part that
 * is not enabled) and the common point_step. PWPP_ERR_INVALID_ARG when no call is bound or packed records are not enabled. */
#define PWPP_OFFSETS_OUT_OF_RANGE 5   /* d_status[f]: d_offsets[f], d_offsets[f + 1] not 0 <= lo <= hi <= capacity; empty frame */
int pwpp_bind_call_packed(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* base, const pwpp_point_layout* layout,
                          int64_t capacity /* records at base */, const int64_t* max_n, const int64_t* d_offsets /* device [nframes + 1] */,
                          const int32_t* d_actions /* NULL: all RUN */);

/* A stream table for a bound call: which sensor stream each frame position serves, read on the GPU at every run or replay, so
 * one bound call (and one captured graph) serves more streams than it has frames, picked per tick by a scheduler on the GPU.
 *
 * pwpp_bind_stream_table: enables the table for the bound call, whichever bind made it (plain, actions, rings or packed). From
 * then on every run or replay reads frame f's stream from d_streams[f], a device int32 array of nframes entries.
 *   - Runs stay the bind's. The runs are still those of the bound streams (maximal groups of consecutive positions with
 *     pairwise distinct streams): they fix the launch sequence, the grids and the scratch slots. Bind distinct streams (for
 *     example 0..F-1) for one run; bind a shape with a repeat (for example [0..63, 0..31]) for two runs, room for a backlog.
 *     The bound stream values matter only for this shape.
 *   - Reading. The run's first kernel reads each entry once into a copy the ctx owns (pwpp_bound_call_streams); the later
 *     kernels read the copy. Frame f's parameter set is stream_set[d_streams[f]], taken on the GPU from a copy of the ctx's
 *     stream-to-set map made at enable time.
 *   - Validation (a replay cannot return an error). s < 0 is a hole: the frame is skipped with PWPP_FRAME_SKIPPED, exactly as
 *     an action SKIP. s >= num_streams: skipped, PWPP_STREAM_OUT_OF_RANGE. Two frames of one run that would run and name the
 *     same stream: the lowest position runs, the others are skipped with PWPP_STREAM_DUPLICATE; frames skipped by their action
 *     claim nothing. A skipped frame goes to its scratch slot as an action SKIP does: no real stream is written and a RESET on
 *     it does not apply.
 *   - Precedence: the action (SKIP or an invalid action), then the stream (hole, out of range, duplicate), then the ring slot
 *     or the packed offsets, then the count. A frame rejected by its action or its stream reads no slot, offset or count.
 *   - Resets. RESET frames of the first run are reset in the table kernel; before every later run a reset launch treats all
 *     of that run's RESET frames as repeats of an earlier run's stream. So pwpp_launch_count rises, over the same call bound
 *     without actions, by exactly runs - 1 per run or replay when actions and a stream table are both bound (the same count as
 *     with actions alone: every later run of a bind already repeats a stream), and a stream table without actions adds nothing.
 *   - Getter rows (PWPP_GETTER_STATE) follow the stream each frame read: for a frame skipped by its action or as a duplicate,
 *     its stream's state after the frame's run; for a hole or an out-of-range id the row is not written. Every other result
 *     (indices, offsets, status, records, xyz, packed results) is indexed by position, as without a table.
 *   - Host getters. pwpp_copy_bin_results fetches the sets the run used from the device with its first copy after a run; a
 *     frame rejected with an invalid id reports the set of its bound stream. The fp32 binning filter is used for a run only
 *     when every set of the ctx allows it (both binning paths are exact: results do not change).
 *   - Identity. d_streams[f] == streams[f] for every f gives the results of the same bind without a table, bit for bit.
 *   - Enable-time work. Enabling is host work that synchronizes and must come before the bound call's first run (capture
 *     included): it grows the state and history buffers by the scratch slots (the longest run) if actions did not already,
 *     and those must not move under a captured graph. PWPP_ERR_INVALID_ARG for no bound call, NULL d_streams, a second enable
 *     or an enable after a run; the bound call is then unchanged. pwpp_unbind_call releases the table.
 *   - Memory: 4 bytes per frame for the copy, 8 bytes per stream for the claim table and the set map.
 *
 * pwpp_bound_call_streams: host-only. The ctx's copy of the streams the last run read, device int32[nframes] at a fixed address
 * while the call stays bound (invalid values included); -1 everywhere before the first run. PWPP_ERR_INVALID_ARG when no call
 * is bound or it has no stream table. */
#define PWPP_STREAM_OUT_OF_RANGE 6   /* d_status[f]: d_streams[f] >= num_streams; the frame was skipped */
#define PWPP_STREAM_DUPLICATE 7      /* d_status[f]: an earlier frame of the same run names the same stream; skipped */
int pwpp_bind_stream_table(pwpp_ctx* ctx, const int32_t* d_streams /* device int32[nframes] */);
int pwpp_bound_call_streams(pwpp_ctx* ctx, const int32_t** d_streams_read);
int pwpp_run_bound_call(pwpp_ctx* ctx, void* cuda_stream);
int pwpp_bound_call_results(pwpp_ctx* ctx, const int32_t** d_indices, const int64_t** d_offsets, const int32_t** d_num_ground,
                            const int32_t** d_status);
#define PWPP_PART_GROUND 1
#define PWPP_PART_NONGROUND 2
int pwpp_bind_record_results(pwpp_ctx* ctx, int parts /* PWPP_PART_* bits: 1, 2 or 3 */);
int pwpp_bound_record_results(pwpp_ctx* ctx, const void** d_ground, const void** d_nonground, const int64_t** h_offsets,
                              const int32_t** d_counts);
int pwpp_bind_packed_xyz(pwpp_ctx* ctx, int parts /* PWPP_PART_* bits: 1, 2 or 3 */);
int pwpp_bound_packed_xyz(pwpp_ctx* ctx, const float** d_ground, const float** d_nonground, const int64_t** d_ground_off,
                          const int64_t** d_nonground_off);
int pwpp_bind_packed_records(pwpp_ctx* ctx, int parts /* PWPP_PART_* bits: 1, 2 or 3 */);
int pwpp_bound_packed_records(pwpp_ctx* ctx, const void** d_ground, const void** d_nonground, const int64_t** d_ground_off,
                              const int64_t** d_nonground_off, int32_t* point_step);

/* Getter results of the bound call: what the reference's other getters return (getGround / getNonground, getCenters /
 * getNormals, getHeight and the adaptive thresholds, H:154-163), at fixed device addresses, for a graph whose next stage takes
 * float32 xyz, the patch planes or the sensor height without a host round trip. Every value is one a host getter returns.
 *
 * pwpp_bind_getter_results: enables them for the bound call. what is a bit set of PWPP_GETTER_GROUND_XYZ,
 * PWPP_GETTER_NONGROUND_XYZ and PWPP_GETTER_STATE, in [1, 7]. Host work like pwpp_bind_record_results (it reserves the buffers,
 * then synchronizes), so it is not capturable; graphs captured before it do not write these results. PWPP_ERR_INVALID_ARG when
 * no call is bound, for what outside [1, 7], and when they are already enabled (one setting per bind: pwpp_unbind_call releases
 * the buffers, and a later bind starts with them off).
 *
 * pwpp_bound_getter_results: host-only; fills *out with fixed device pointers (PWPP_ERR_INVALID_ARG when no call is bound).
 *   - xyz: ground_xyz and nonground_xyz are float32 rows of 3 (NULL for a part that is not enabled), sum(max_n) rows each.
 *     Frame f's rows start at row h_row_off[f] of both (host int64[nframes + 1], the prefix sum of max_n). xyz_counts is
 *     device int32[2 nframes]: ground count, then non-ground count of every frame (NULL when no xyz part is enabled). Row k of a
 *     part is row k of pwpp_copy_ground_xyz / pwpp_copy_nonground_xyz of that frame after the same run, bit for bit, in the list
 *     order the call was bound with (for an RNR-rejected point, its original z). Rows past a count are never written; a
 *     skipped frame or one whose count or slot was out of range has counts 0.
 *   - Patches: centers and normals (float32 rows of 3), num_patches (device int32[nframes]) and patch_row_stride. Frame f's
 *     num_patches[f] rows start at row f * patch_row_stride, bit for bit what pwpp_copy_centers / pwpp_copy_normals return.
 *     They are k_gle's own output: always available while a call is bound, with no enable bit and no launch.
 *   - State: states is device pwpp_state[nframes] (NULL when not enabled). Row f is the state of frame f's stream immediately
 *     after frame f: what pwpp_get_state on that stream would return had the call stopped there. A skipped frame (SKIP or an
 *     invalid action) gets its stream's state as its earlier frames of the call left it (the real stream, never a scratch
 *     slot); an out-of-range count or slot, the state after the empty frame; a RESET frame, the state after the reset and then
 *     the frame. A stream bound twice (a backlog) has two rows that differ as after two direct calls.
 * Rules:
 *   - Valid until the next call or replay. Direct calls between runs never write the xyz or state buffers; they do overwrite
 *     the patch rows and counts, like the index lists.
 *   - pwpp_launch_count rises, per pwpp_run_bound_call, by one xyz gather launch when either xyz part is enabled (after the
 *     last run's output kernel, also when every max_n is 0), and by one state launch after each run of the call (a run: a
 *     maximal group of consecutive frames with pairwise distinct streams) when the state is enabled. Nothing for the patches.
 *   - Memory: 12 sum(max_n) bytes per enabled xyz part plus 8 nframes bytes of counts and 8 (nframes + 1) bytes of row
 *     offsets when either is enabled, and sizeof(pwpp_state) nframes bytes for the state. */
#define PWPP_GETTER_GROUND_XYZ 1
#define PWPP_GETTER_NONGROUND_XYZ 2
#define PWPP_GETTER_STATE 4
typedef struct pwpp_bound_getters {
  const float* ground_xyz;        /* device float32 [sum(max_n)][3], or NULL */
  const float* nonground_xyz;     /* device float32 [sum(max_n)][3], or NULL */
  const int64_t* h_row_off;       /* host int64 [nframes + 1]: frame f's rows start at row h_row_off[f] */
  const int32_t* xyz_counts;      /* device int32 [nframes][2]: ground, non-ground; NULL without an xyz part */
  const float* centers;           /* device float32 rows of 3: frame f's patches start at row f * patch_row_stride */
  const float* normals;
  const int32_t* num_patches;     /* device int32 [nframes] */
  int64_t patch_row_stride;
  const pwpp_state* states;       /* device [nframes], or NULL */
} pwpp_bound_getters;
int pwpp_bind_getter_results(pwpp_ctx* ctx, int what /* PWPP_GETTER_* bits, 1..7 */);
int pwpp_bound_getter_results(pwpp_ctx* ctx, pwpp_bound_getters* out);
/* Releases the bound call, its record results and its getter results (PWPP_ERR_INVALID_ARG when none is bound). Its index results stay readable
 * until the next call. */
int pwpp_unbind_call(pwpp_ctx* ctx);

/* ---- several bound calls: one captured graph per batch shape over the same sensor streams ----------------------------------
 * A pipeline that replays CUDA graphs captures one graph per batch shape and picks one per step (a bucket ladder of 1, 4, 16
 * and 64 frames), or keeps a ring-bound live graph beside a packed graph of logged scans. A ctx holds bound calls 0 ..
 * PWPP_MAX_BOUND_CALLS - 1, each with its own shape (frames, capacities, bind kind, runs), over the ctx's one set of streams.
 *
 * pwpp_select_bound_call: selects bound call k. Host-only: no synchronisation and no launch. k outside
 * [0, PWPP_MAX_BOUND_CALLS) returns PWPP_ERR_INVALID_ARG and the selection is unchanged. Call 0 is selected when the ctx is
 * created, so a caller that never selects has the one bound call described above.
 * pwpp_selected_bound_call: the selected call (PWPP_ERR_INVALID_ARG for a NULL ctx).
 *
 * Every bind (pwpp_bind_call, _actions, _rings, _packed), pwpp_bind_stream_table, pwpp_bind_record_results,
 * pwpp_bind_getter_results, pwpp_bind_packed_xyz, pwpp_bind_packed_records, pwpp_run_bound_call, every pwpp_bound_* getter and
 * pwpp_unbind_call act on the selected call, with the semantics above. A bind on a selected call that is already bound returns
 * PWPP_ERR_INVALID_ARG ("already bound"). A graph captured from pwpp_run_bound_call holds the call selected at capture: a
 * later selection has no effect on it.
 *
 * Rules:
 *   - Shared. All bound calls share the stream states and histories, the parameter sets, the output order, the scratch state
 *     slots (as many as the longest run of any call) and the work buffers. So the caller orders runs and replays of different
 *     calls as it orders direct calls: on one CUDA stream, or with its own events. Replays of two bound calls of one ctx at the
 *     same time are not supported.
 *   - Per call. Each call has its own device tables and status array, its copies of the actions, ring slots and streams, the
 *     claim table of its stream table, and its record, getter (xyz and state), packed-xyz and packed-record buffers. They hold
 *     that call's last run until its next run: runs of other calls and direct calls never write them. The index results
 *     (d_indices, d_offsets, d_num_ground of pwpp_bound_call_results) and the patch rows of pwpp_bound_getter_results live in
 *     the work buffers: they hold the last run of any call (or the last direct call).
 *   - Growth. A bind may need larger work buffers (sum(max_n) points, nframes frames; under PWPP_ORDER_REFERENCE_EXACT also the
 *     fix-up's scratch, under PWPP_ARITH_REFERENCE the fit scratch) and a bind with actions or a stream-table enable more scratch slots. Before any bound call has run or
 *     been captured they grow as needed. Afterwards captured graphs hold them, so such a bind or enable returns
 *     PWPP_ERR_CAPACITY before anything changes; the message names the points and frames or the scratch slots it needs. To
 *     avoid it, bind every call, widest shape first (each buffer then grows once), and enable its tables before the first run
 *     or capture. Creating the
 *     ctx with a large enough max_points_per_frame pre-sizes the work buffers, not the scratch slots: only binds make those.
 *   - Freeze. The freeze of the work buffers holds while any call is bound: a direct call that would grow a buffer returns
 *     PWPP_ERR_CAPACITY, pwpp_set_output_order and pwpp_clone return PWPP_ERR_INVALID_ARG. pwpp_unbind_call releases only the
 *     selected call; it moves no shared buffer, so the graphs of the other calls stay valid.
 *   - Host getters follow the last call: the bound call whose pwpp_run_bound_call or pwpp_bound_call_results came last, not
 *     the selected one. Unbinding it leaves its index results readable until the next call. A bind ends the last call's
 *     results, as with one bound call.
 *   - pwpp_launch_count rises per run exactly as for the same call bound alone in a fresh ctx.
 *   - Memory: each bound call's own tables and result buffers, as described for its bind; nothing else per call. */
#define PWPP_MAX_BOUND_CALLS 32
int pwpp_select_bound_call(pwpp_ctx* ctx, int k);
int pwpp_selected_bound_call(const pwpp_ctx* ctx);

/* ---- width ladders: the GPU picks how many positions a bound call launches, at every run or replay ----------------------------
 * A scheduler kernel inside the caller's graph that picks the streams of a tick (a stream table) cannot tell the host how many
 * sensors arrived without a device-to-host read, so it cannot pick one of several graphs. A width ladder lets one graph do it:
 * at every run or replay the GPU reads the table kernel's status array and launches the call cut to the narrowest width of the
 * ladder that holds every position that runs. A narrow width sizes every grid for the capacities of its first positions only.
 * The kernel variants stay those of each run's full length: a 4-wide launch of a 64-frame run keeps the batch kernels, because
 * the small-call kernels (PWPP_SMALL_CALL) give plane fits that differ from the batch kernels' in the last bits, which moves the
 * adaptive thresholds, and a ladder changes no result.
 *
 * pwpp_bind_width_ladder: enables the ladder for the selected bound call. widths[0 .. nwidths) must be strictly increasing and
 * each in [1, nframes); the call's own nframes is always the implicit last width, so 1 <= nwidths <= PWPP_MAX_LADDER_WIDTHS - 1.
 * Host work that synchronizes: it captures the call's launch sequence cut
 * at every width into graphs the call owns, so later result enables (pwpp_bind_record_results, pwpp_bind_getter_results,
 * pwpp_bind_packed_xyz, pwpp_bind_packed_records) and pwpp_bind_stream_table on that call return PWPP_ERR_INVALID_ARG: enable
 * them before the ladder. It grows no buffer, so it is allowed after runs and captures; graphs captured before it keep running
 * without the ladder. Once enabled, the call counts as captured for the growth rule of "Several bound calls".
 * PWPP_ERR_INVALID_ARG, with the call unchanged, when no call is bound, for bad widths (NULL, nwidths outside that range, not
 * strictly increasing, outside [1, nframes)), for a second enable, and for a call with neither actions nor a
 * stream table (every position of such a call runs, so the widest width would always be chosen). pwpp_unbind_call releases it.
 *
 * The width rule. A position RUNS when the table kernel leaves it status 0, PWPP_COUNT_OUT_OF_RANGE, PWPP_SLOT_OUT_OF_RANGE or
 * PWPP_OFFSETS_OUT_OF_RANGE (frames whose stream state advances). It is REJECTED when its status is PWPP_FRAME_SKIPPED,
 * PWPP_ACTION_INVALID, PWPP_STREAM_OUT_OF_RANGE or PWPP_STREAM_DUPLICATE. With L = 1 + the last position that runs (0 when none
 * does), the run launches the smallest ladder width w >= max(L, 1). A scheduler that compacts the present streams to the
 * front gets the narrow launch; one that leaves a present stream at the last position gets the full width.
 *
 * The contract: enabling a ladder changes no result. After every run or replay, everything equals, bit for bit, what the same
 * call without a ladder gives after the same runs: the indices, offsets, num_ground, status and the read copies of streams,
 * slots and actions; the record, getter (xyz and state rows), packed-xyz and packed-record buffers, including the bytes past
 * every count, which stay unwritten; the patch rows; everything the host getters return (indices, xyz, centers, normals, bin
 * results, bin ids, per-frame state); and the export blob of every stream. The positions at or past w are rejected frames: they
 * still run, as the empty frames on their scratch slots that they are without a ladder, through the same kernels with grids
 * sized for empty frames, and the gathers still cover all nframes positions.
 *
 * Graphs. A run on a stream that is capturing (global capture mode included) adds to the caller's graph the table kernel,
 * k_ladder_select and one conditional SWITCH node whose bodies are copies of the prebuilt width graphs; an uncaptured run
 * launches the same graph, built at enable time, as an executable graph the call owns. CUDA's rules for graphs that contain a
 * conditional node apply to the caller's graph: it cannot be cloned, cannot be used as a child graph node, and one executable
 * instance of it must not run twice at once. A caller that embeds its graph as a child graph uses the call without a ladder.
 *
 * pwpp_launch_count rises per run exactly as for the same call without a ladder, plus one for the selector, whatever width runs.
 *
 * pwpp_bound_call_width: host-only. *d_width is a device int32 at a fixed address while the call stays bound: the width the last
 * run or replay launched. For a call without a ladder it holds nframes; a ladder enable sets it to 0 until its first run.
 * PWPP_ERR_INVALID_ARG when no call is bound.
 *
 * Memory: 4 bytes of device memory per bound call for the width, and per ladder one graph per width. */
#define PWPP_MAX_LADDER_WIDTHS 8
int pwpp_bind_width_ladder(pwpp_ctx* ctx, int nwidths, const int32_t* widths);
int pwpp_bound_call_width(pwpp_ctx* ctx, const int32_t** d_width);

/* cudaDeviceSynchronize() on the ctx's device: what a binding calls before handing device memory produced on an unknown
 * stream to pwpp_estimate_device (and what makes its results visible to every stream afterwards). */
int pwpp_device_synchronize(pwpp_ctx* ctx);
int pwpp_synchronize(pwpp_ctx* ctx);

/* ---- results of the last estimate call, per frame f (position in the call) -------------- */

/* getGroundIndices / getNongroundIndices (H:159-160, S:18-26): int32 indices into the frame's
 * point array. Every input point appears in exactly one of the two lists (S:545-548).
 * Order: concentric-zone emission order of the reference (S:184-311) at bin granularity;
 * within one bin ascending point index (the reference's within-bin order is z-sorted with
 * implementation-defined ties, S:199). */
int64_t pwpp_num_ground(pwpp_ctx* ctx, int f);
int64_t pwpp_num_nonground(pwpp_ctx* ctx, int f);
int pwpp_copy_ground_indices(pwpp_ctx* ctx, int f, int32_t* dst);
int pwpp_copy_nonground_indices(pwpp_ctx* ctx, int f, int32_t* dst);
/* getGround / getNonground (H:157-158, S:8-16): row-major n x 3 float xyz of the listed points
 * (for RNR-rejected points the original z, S:393). */
int pwpp_copy_ground_xyz(pwpp_ctx* ctx, int f, float* dst);
int pwpp_copy_nonground_xyz(pwpp_ctx* ctx, int f, float* dst);
/* getCenters / getNormals (H:162-163, S:211-212): one row per bin that was plane-fitted
 * (>= num_min_pts points), in (zone, ring, sector) order; row-major k x 3 float. */
int pwpp_num_patches(pwpp_ctx* ctx, int f);
int pwpp_copy_centers(pwpp_ctx* ctx, int f, float* dst);
int pwpp_copy_normals(pwpp_ctx* ctx, int f, float* dst);
/* getHeight (H:154): the ADAPTIVE sensor height of STREAM f after its last frame (S:348). */
double pwpp_height(pwpp_ctx* ctx, int f);
/* getTimeTaken (H:155): microseconds of the last estimate call (whole call, all frames). */
double pwpp_time_us(pwpp_ctx* ctx);
/* Device-side split of that time for the last pwpp_estimate_host call, when the call ran as one chunk on one stream (calls of
 * a few frames — the reference's one-frame-per-call pattern): out = { host->device copy, kernels, device->host copy, all three }
 * in microseconds, from CUDA events on the call's stream. pwpp_time_us minus out[3] is host-side overhead. */
int pwpp_call_times_us(pwpp_ctx* ctx, float out[4]);

/* Device-side view of the index lists of the last call (zero-copy consumers, benchmark):
 * *d_indices -> int32 array laid out like the input (frame f's region starts at its point
 * offset); inside a region the ground list comes first, then the nonground list.
 * *d_num_ground -> int32[nframes]. Valid until the next estimate call. */
int pwpp_device_results(pwpp_ctx* ctx, const int32_t** d_indices, const int32_t** d_num_ground);

/* Order of the points INSIDE a bin's contribution to the index lists (the order of the bins, of the RNR / out-of-range
 * prefix and of the TGR-reverted patches is always the reference's, S:264-304):
 *   PWPP_ORDER_BIN        ascending point index (default of the C-ABI: what the fit kernels produce, no extra work);
 *   PWPP_ORDER_REFERENCE  the reference's order: ground part in ascending z; non-ground part = R-VPF removals by iteration,
 *                         each in ascending z, then the final rejects in ascending z (S:199, S:495-504, S:529-541); equal z
 *                         in ascending point index (= the reference with a stable per-bin sort). One extra kernel (a sort of
 *                         every fitted patch). The drop-in C++ class and pypatchworkpp select it by default.
 *   PWPP_ORDER_REFERENCE_EXACT  the unmodified reference's lists: as PWPP_ORDER_REFERENCE, with equal z in the order the
 *                         reference's std::sort leaves them as built by libstdc++ (GCC's introsort; not libc++'s or MSVC's).
 *                         Whenever the label sets are identical to the reference's, the lists are identical element for
 *                         element. A fix-up kernel per patch-size class runs after the sort: pwpp_launch_count rises by five
 *                         per launch range over PWPP_ORDER_REFERENCE (one per class, on that class's stream); patches without
 *                         two equal z in one part leave it at once. Patches above 512 points use a scratch of 16 bytes per
 *                         point of the call, reserved with the work buffers (so a bound call reserves it at bind).
 * Takes effect with the next estimate call. A bound call keeps the order it was bound with. */
#define PWPP_ORDER_BIN 0
#define PWPP_ORDER_REFERENCE 1
#define PWPP_ORDER_REFERENCE_EXACT 2
int pwpp_set_output_order(pwpp_ctx* ctx, int order);
/* Counters of the PWPP_ORDER_REFERENCE_EXACT fix-up since the context was created or the last reset: out[0] = patches with a
 * tie in z inside one part (their libstdc++ order simulated), out[1] = segments sorted by the depth-limit heap sort, out[2] =
 * bins holding a NaN z (std::sort run literally in one thread). Synchronises the device; reset != 0 zeroes them afterwards. */
int pwpp_order_exact_counts(pwpp_ctx* ctx, uint64_t out[3], int reset);

/* Arithmetic of the plane fits and of A-GLE (pwpp_set_arithmetic; the default is PWPP_ARITH_DOUBLE).
 *   PWPP_ARITH_DOUBLE     the reference's formulas in IEEE double with order-free sums and a closed-form eigen solve: index
 *                         SETS equal the reference's except where fp32 rounding decides a point (DESIGN.md section 3).
 *   PWPP_ARITH_REFERENCE  the reference's own arithmetic (S:47-75, S:217-223, S:551-554), so every result is the reference
 *                         build's bit for bit, patches of 1-4 points, collinear and vertical patches included:
 *       - every plane fit sums its point set sequentially in fp32 in the z-sorted order of the bin (mean: 3 sums divided by
 *         (float) n; covariance: 6 sums of (q_i - mean_i) * (q_j - mean_j) divided by (float) (double) (n - 1)), then runs the
 *         fp32 two-sided Jacobi SVD with the sign flip of the normal; d = -(x0 + (x1 + x2)) in fp32. Every operation is
 *         separately rounded. The point sets are the reference's subsequences of the sorted bin (R-VPF seeds and kept points,
 *         R-GPF seeds and each round's kept points). Equal z follow the output order's build: under PWPP_ORDER_BIN and
 *         PWPP_ORDER_REFERENCE ascending point index (std::stable_sort: results bit for bit libpwref_stable.so's), under
 *         PWPP_ORDER_REFERENCE_EXACT the order libstdc++'s std::sort leaves them in (results bit for bit the unmodified
 *         reference's, libpwref.so). So in a bin with equal z the output order can change the planes, and with them the
 *         labels, in the low bits where the two builds differ;
 *       - the point-plane distance is ((n0 x + n1 y) + n2 z) in fp32 plus d in double; the LPR height is the double sum of
 *         at most num_lpr floats in sorted order;
 *       - A-GLE reads the fp32 plane: flatness is the fp32 minimum of the singular values, line_variable the fp32 quotient
 *         sv0 / sv1 and heading the double sum of fp32 products mean_i * normal_i. The thresholds, sensor_height and the
 *         histories follow from the same sequential double sums as in the default mode;
 *       - patch records, centers and normals hold the float values (widened where the record is double). TGR's double exp
 *         may differ from glibc's in the last bit; it only feeds the > 0.5 revert test.
 *     Unchanged: the two defined deviations (history bound, patches without a plane), non-finite z, RNR, binning and the
 *     gate. pwpp_launch_count rises exactly as in the default mode (one fit kernel per patch-size class, one k_gle).
 *     A fit of the reference mode costs sequential fp32 chains over its point set: the largest patch of a call bounds its
 *     fit stage (DESIGN.md section 3 gives the measured cost). Memory: the work buffers of the mode grow by 46 bytes per point
 *     of the call (sort keys 16, staged points 16, fit set 12, flags 2), the storage of the patches above 512 / 2048 points
 *     that do not fit the fit kernels' shared memory, each patch at its own offset (about 5.5 GB for a call of 120 M points);
 *     a bind in this mode reserves them as well.
 * Rules, as for pwpp_set_output_order: refused (PWPP_ERR_INVALID_ARG) while any call is bound, so a captured graph keeps the
 * arithmetic it was bound with; pwpp_clone copies it; stream-state blobs have one format in both modes and move between
 * them. Switching back to PWPP_ARITH_DOUBLE gives exactly the results of a context that never left it.
 * pwpp_arithmetic returns the context's mode (PWPP_ERR_INVALID_ARG for a NULL ctx). */
#define PWPP_ARITH_DOUBLE 0
#define PWPP_ARITH_REFERENCE 1
int pwpp_set_arithmetic(pwpp_ctx* ctx, int arith);
int pwpp_arithmetic(const pwpp_ctx* ctx);

/* Host-side zero-copy view of the index lists of the last call (batch consumers: the per-frame getters above copy each
 * list once more, which for a 1024-frame batch is 0.5 GB of host memcpy): *h_indices -> the page-locked int32 buffer the
 * device lists were copied into, laid out like pwpp_device_results (frame f's region starts at point offset
 * *h_offsets[f]: ground list, then nonground list); *h_num_ground -> int32[nframes]. Fetches the lists from the device
 * if the call was a device-input call. Valid until the next estimate call. */
int pwpp_host_results(pwpp_ctx* ctx, const int32_t** h_indices, const int32_t** h_num_ground, const int64_t** h_offsets);

/* Placement helper for multi-GPU hosts: binds the CALLING THREAD (and with it the page-locked buffers it allocates
 * afterwards: first touch) to the CPUs of the NUMA node the device hangs off (sysfs numa_node / cpulist of its PCI
 * function). Returns the node (>= 0), or -1 if the topology could not be read (nothing changed). Call it before
 * pwpp_host_alloc / pwpp_create in a one-process-per-GPU launch. */
int pwpp_bind_host_to_device(int device);

/* ---- per-bin diagnostics for parity tests (not part of the reference surface) ------------ */

/* Per-bin record of the last call, frame f: bin ids in (zone,ring,sector) order. */
typedef struct pwpp_bin_result {
  double mean[3];      /* pc_mean_          (S:59-60) */
  double normal[3];    /* normal_, z >= 0   (S:66-68) */
  double sv[3];        /* singular_values_, descending (S:63) */
  double d;            /* d_                (S:74)    */
  int32_t n;           /* points binned into the patch (S:602-614) */
  int32_t n_ground;    /* |regionwise_ground_| (S:530)                 */
  int32_t verdict;     /* see PWPP_VERDICT_*                           */
  int32_t fitted;      /* 1 if n >= num_min_pts (S:191)                */
} pwpp_bin_result;

#define PWPP_VERDICT_SKIPPED 0        /* < num_min_pts: all nonground (S:191-195)  */
#define PWPP_VERDICT_NOT_UPRIGHT 1    /* S:262-265 */
#define PWPP_VERDICT_FAR_GROUND 2     /* S:266-269 */
#define PWPP_VERDICT_HEADING 3        /* S:270-273 */
#define PWPP_VERDICT_NEAR_GROUND 4    /* S:274-277 */
#define PWPP_VERDICT_TGR_REVERTED 5   /* S:444-450 */
#define PWPP_VERDICT_TGR_REJECTED 6   /* S:452-458, or enable_TGR == false (S:297-299) */

int pwpp_copy_bin_results(pwpp_ctx* ctx, int f, pwpp_bin_result* dst /* [nbins of frame f's set, <= pwpp_num_bins] */);
/* Polar bin id of every point of frame f as computed by the binning kernel:
 * 0..nbins-1, or nbins (= RNR hit, S:391-396) or nbins+1 (= outside (min_range,max_range], S:617-619). */
int pwpp_copy_bin_ids(pwpp_ctx* ctx, int f, uint16_t* dst /* [n_f] */);

/* ---- measurement hooks (not part of the reference surface) ---------------------------------- */

/* Page-locked host memory for callers that have no CUDA binding of their own. pwpp_estimate_host copies
 * straight from a caller buffer that is page-locked (allocated here, by cudaHostAlloc or registered with
 * cudaHostRegister) and row-major N x 4; any other buffer is first staged through the ctx's pinned buffer. */
void* pwpp_host_alloc(size_t bytes);
void pwpp_host_free(void* p);

#define PWPP_NUM_STAGES 11  /* bin_hist, bin_scan, scatter, fit_S, fit_L3, fit_L2, fit_L1, fit_M, fit_X, gle, emit */
/* With profiling on, CUDA events are recorded around every kernel of the following estimate calls;
 * pwpp_stage_times_ms() synchronizes and returns the device time of each stage of the LAST call. */
int pwpp_set_profiling(pwpp_ctx* ctx, int enabled);
int pwpp_stage_times_ms(pwpp_ctx* ctx, float* ms /* [PWPP_NUM_STAGES] */);
const char* pwpp_stage_name(int stage);
/* Number of kernels this ctx has launched since creation. */
int64_t pwpp_launch_count(const pwpp_ctx* ctx);

/* ---- temporal state (S:338-375), per STREAM f --------------------------------------------- */

int pwpp_get_state(pwpp_ctx* ctx, int f, pwpp_state* out);
/* Histories: ring r of update_elevation_ / update_flatness_ (H:174-175); dst holds n_* doubles. */
int pwpp_copy_history(pwpp_ctx* ctx, int f, int ring, int which /*0=elevation,1=flatness*/, double* dst);
/* Checkpoint / migration of one stream (SURVEY.md 8f-4): the COMPLETE temporal state the reference object carries from
 * frame to frame — adaptive sensor height and thresholds (S:347-350, S:368), both history arrays (H:174-175) and the
 * plane members left by the last estimate_plane call (S:49 keeps them when a patch's seed set is empty) — as one
 * opaque blob. A blob exported from stream f of one ctx can be imported into any stream of any ctx created with the
 * same parameters (another GPU, another process, a later run): the next frame then gives bit-identical results.
 * pwpp_export_state synchronizes with the last estimate call; pwpp_import_state takes effect before the next one. */
size_t pwpp_state_blob_size(const pwpp_ctx* ctx);           /* the largest over the sets: fits any stream's blob */
size_t pwpp_stream_state_blob_size(const pwpp_ctx* ctx, int s); /* the blob of stream s (its set's hist_cap); 0 for a bad s */
int pwpp_export_state(pwpp_ctx* ctx, int f, void* blob /* [pwpp_state_blob_size] */);
int pwpp_import_state(pwpp_ctx* ctx, int f, const void* blob, size_t bytes);

/* ---- stream state on the GPU: snapshot, restore and fork streams inside the caller's CUDA graph --------------------------
 * pwpp_export_state / pwpp_import_state move one stream per call through host memory and synchronize. These two move any list
 * of streams between the ctx and a device buffer of blob rows, enqueued on a CUDA stream with no host synchronization, so a
 * graph can snapshot its streams before a tick and roll some of them back after it on a decision made on the GPU (a check
 * that rejects a frame, a sensor fault, a replayed segment), fork a stream into another, or hand 64 sensors to another ctx.
 *
 * pwpp_export_states_device: for entry i of the device list d_streams (int32[n]), the complete state of stream
 * s = d_streams[i] into row i of d_blobs, which starts at byte i * blob_stride. The row is byte for byte what
 * pwpp_export_state writes for s (pwpp_stream_state_blob_size(ctx, s) bytes: header, state with the carried plane, the eight
 * history rows of s's set); bytes of the row past that size are never written. d_status[i] = PWPP_STATE_OK, or
 * PWPP_STATE_SKIPPED for s < 0 and PWPP_STATE_OUT_OF_RANGE for s >= num_streams, whose rows are not written.
 *
 * pwpp_import_states_device: the reverse copy, row i into stream d_streams[i], with the checks of pwpp_import_state made on the
 * GPU. A replay cannot return an error, so every entry gets a status in d_status[i]:
 *   - PWPP_STATE_OK: the stream now holds the row's state.
 *   - PWPP_STATE_SKIPPED: d_streams[i] < 0; nothing is read or written. A graph decides on the GPU which streams to restore by
 *     writing -1 into the entries it leaves alone.
 *   - PWPP_STATE_OUT_OF_RANGE: d_streams[i] >= num_streams. Only streams [0, num_streams) are reachable, never the scratch
 *     slots of bound calls with actions.
 *   - PWPP_STATE_BLOB_MISMATCH: the row's header is not one pwpp_import_state accepts for that stream (magic, PWPP_ABI_VERSION,
 *     the history capacity of the stream's set, the state size); the stream is untouched.
 *   - PWPP_STATE_DUPLICATE: an earlier entry of the call names the same stream; the first entry wins, whatever its status.
 *
 * Rules, for both:
 *   - Capturable. No host synchronization, no allocation, no host-memory copy: kernels only, enqueued on cuda_stream (NULL =
 *     the ctx's own stream), which may be capturing. The stream ids are read on the GPU when the launch runs, so a graph
 *     replays with the ids the list holds at that moment; each entry reads its id once.
 *   - Ordering is the caller's, as for pwpp_run_bound_call: calls of this ctx on other streams are not waited for. The host
 *     getters, pwpp_get_state and pwpp_export_state see a device import once the caller has synchronized cuda_stream.
 *   - Buffer moves. A captured graph holding these calls stays valid until the ctx's state buffers move, which only a bind
 *     with actions may do (it grows them by its scratch slots, see pwpp_bind_call_actions): bind first, then capture.
 *   - Host checks, before anything is launched (PWPP_ERR_INVALID_ARG): n outside [0, 65535]; NULL d_streams or d_blobs with
 *     n > 0; blob_stride below pwpp_state_blob_size(ctx) or not a multiple of 16; d_blobs not 16-byte aligned. n == 0
 *     launches nothing. d_status may be NULL (not written).
 *   - pwpp_launch_count rises by 1 per export and by 2 per import (a claim launch that resolves duplicates, then the copy).
 *   - Interop. A row copied to the host is a valid pwpp_import_state blob, and a pwpp_export_state blob copied into a row is
 *     a valid row. The blob format is the one of pwpp_export_state.
 *   - Memory: 8 num_streams bytes on the device for every ctx (the claim table, -1 between calls, and the history capacity of
 *     every stream). */
#define PWPP_STATE_OK 0
#define PWPP_STATE_SKIPPED 1         /* d_status[i]: d_streams[i] < 0; nothing read or written */
#define PWPP_STATE_OUT_OF_RANGE 2    /* d_status[i]: d_streams[i] >= num_streams */
#define PWPP_STATE_BLOB_MISMATCH 3   /* d_status[i]: the row's header does not fit the stream; the stream is untouched */
#define PWPP_STATE_DUPLICATE 4       /* d_status[i]: an earlier entry of the call names the same stream */
int pwpp_export_states_device(pwpp_ctx* ctx, int n, const int32_t* d_streams, void* d_blobs, int64_t blob_stride,
                              int32_t* d_status /* NULL: not written */, void* cuda_stream);
int pwpp_import_states_device(pwpp_ctx* ctx, int n, const int32_t* d_streams, const void* d_blobs, int64_t blob_stride,
                              int32_t* d_status /* NULL: not written */, void* cuda_stream);

/* A copy of a whole ctx, what `PatchWorkpp b = a;` is for the reference's value type: a new ctx on `device` (< 0: src's
 * device) with src's parameter sets, stream->set map, num_streams, point capacity and output order, every stream's state
 * and histories, and the results of src's last call. Every per-frame getter answers on the clone as on src (counts, index
 * lists, xyz, centers, normals, num_patches, bin results and ids, pwpp_time_us, pwpp_device_results and pwpp_host_results on
 * the clone's own buffers), and the next frames give bit-identical results on both.
 *   - Host work: synchronizes src, copies device to device (cudaMemcpyPeer when device differs from src's), then synchronizes
 *     the clone. src is not modified.
 *   - PWPP_ERR_INVALID_ARG while src holds a bound call (pwpp_unbind_call first): a bound call's tables point at the caller's
 *     buffers and at graphs, which a copy cannot take over.
 *   - Record results are not carried: on the clone the records getters answer as after a call that took no records.
 *   - The clone's launch count starts at 0 and it holds no bound call; pwpp_destroy releases it like any ctx. */
int pwpp_clone(const pwpp_ctx* src, int device /* < 0: src's device */, pwpp_ctx** out);

/* Re-initialises stream f / all streams to the constructor state (a fresh PatchWorkpp instance).
 * Stream-ordered: enqueued behind the last estimate call, no host synchronization. */
int pwpp_reset_stream(pwpp_ctx* ctx, int f);
int pwpp_reset_all(pwpp_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* PWPP_H_ */
