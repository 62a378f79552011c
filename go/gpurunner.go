//go:build cgo

// Package anomalydetector: GPU job runner behind the function-variable seam of
// pkg/controller/anomalydetector/controller.go:54-59 (see INTEGRATION.md).  This file is the source a Theia
// maintainer drops next to controller.go; it is NOT compiled in this repository (no Go toolchain in the build
// image) -- its behaviour is exercised through the identical Python binding (theia_b200/engine.py,
// theia_b200/controller.py, tests/test_host_mirror.py).
package anomalydetector

/*
#cgo CFLAGS:  -I${SRCDIR}/../../../third_party/theia_tad/include
#cgo LDFLAGS: -L${SRCDIR}/../../../third_party/theia_tad/lib -ltheia_tad -Wl,-rpath,$ORIGIN
#include <stdlib.h>
#include <string.h>
#include "theia_tad.h"
*/
import "C"

import (
	"fmt"
	"sync"
	"sync/atomic"
	"unsafe"
)

// FlowColumns is what the ClickHouse reader hands over: one slice per selected column of default.flows
// (create_table.sh:31-85), IPs already mapped to u32 (IPv4) or dictionary ids.
//
// FlowEnd and Throughput are required.  A key column the job's GROUP BY does not use is left nil (the aggregated-flow
// modes use two or three of the six key slots, anomaly_detection.py:511-609): the engine then treats it as all zero.
// Every non-nil slice must have len(FlowEnd) elements.  SrcNS / DstNS are namespace dictionary ids, needed only
// together with JobSpec.NSIgnore.
type FlowColumns struct {
	SrcIP, DstIP, FlowStart, FlowEnd []uint32
	SrcPort, DstPort                 []uint16
	Proto                            []uint8
	Throughput                       []uint64
	SrcNS, DstNS                     []uint32
}

// JobSpec carries the already validated arguments startSparkApplication would have put into argv
// (controller.go:530-623).
type JobSpec struct {
	Algo       string // EWMA | ARIMA | DBSCAN
	SumReducer bool   // aggregated-flow modes use sum(throughput), per-connection mode max(throughput)
	StartTime  uint32 // epoch seconds, 0 = unbounded; needs FlowColumns.FlowStart (a key column): the modes whose key has
	// no flowStartSeconds (external, svc) apply the lower bound in their SELECT's WHERE clause and pass 0 here
	EndTime  uint32
	ID       string
	NSIgnore []uint32 // --ns-ignore-list (controller.go:546), mapped to the namespace ids used in SrcNS / DstNS
	// rows of the whole table over all ranks when the job runs on several GPUs (world_size > 1); 0 on one GPU
	GlobalRows uint64
}

// AnomalyRow is one row of default.tadetector (create_table.sh:363-384) minus the per-job constants.
type AnomalyRow struct {
	SrcIP, DstIP, FlowStart, FlowEnd  uint32
	SrcPort, DstPort                  uint16
	Proto                             uint8
	StdDev, AlgoCalc, Throughput      float64
}

type gpuJob struct {
	job  *C.tad_job
	cols C.tad_columns
	fed  chan struct{} // StartStream: closed once the feeding goroutine no longer calls into the job (nil for Start)
}

type gpuJobRunner struct {
	ctx    *C.tad_ctx
	jobs   sync.Map    // id -> *gpuJob
	share  atomic.Bool // SetFitSharing turned fit sharing on: StartStream flags its jobs
	beside atomic.Bool // SetFitBeside: Start (StartStream while share is on) flags its ARIMA jobs to fit beside a running fit
	lend   atomic.Bool // SetStreamLend: StartStream flags its jobs to lend the GPU while their SELECT is read
}

func newGPUJobRunner(device int) (*gpuJobRunner, error) {
	cfg := C.tad_config{device: C.int32_t(device), world_size: 1, rank: 0}
	var ctx *C.tad_ctx
	if rc := C.tad_init(&cfg, &ctx); rc != C.TAD_OK {
		return nil, fmt.Errorf("tad_init: %s", C.GoString(C.tad_strerror(rc)))
	}
	return &gpuJobRunner{ctx: ctx}, nil
}

// SetMemoryBudget caps the device memory the runner's context holds (0 = what is free when a job starts, less a
// headroom).  A job larger than the budget runs in hash-range passes instead of failing; it takes effect for jobs that
// start after the call.  The controller sets it once after newGPUJobRunner when the GPU is shared.
func (r *gpuJobRunner) SetMemoryBudget(bytes uint64) error {
	if rc := C.tad_set_memory_budget(r.ctx, C.uint64_t(bytes)); rc != C.TAD_OK {
		return fmt.Errorf("tad_set_memory_budget: %s", C.GoString(C.tad_strerror(rc)))
	}
	return nil
}

// SetHostBudget lets the runner's context pin up to `bytes` of host memory for its host row store (0 = none, the
// default; nonzero values below 64 MiB are refused).  A streamed job that needs several hash-range passes then keeps its
// rows there and StartStream runs its SELECT once; if the store would not hold the rows, the job asks for the rows again
// as without a store.  It takes effect for jobs that start after the call.
func (r *gpuJobRunner) SetHostBudget(bytes uint64) error {
	if rc := C.tad_set_host_budget(r.ctx, C.uint64_t(bytes)); rc != C.TAD_OK {
		return fmt.Errorf("tad_set_host_budget: %s", C.GoString(C.tad_strerror(rc)))
	}
	return nil
}

// SetFitSharing turns fit sharing on with a reserve of `reserve` device bytes (0 = off, the default; nonzero values below
// 64 MiB are refused).  While an ARIMA job fits, a queued EWMA or DBSCAN job then runs in the reserve instead of waiting
// for the whole fit phase, and the ARIMA job plans in the memory budget less the reserve.  Jobs from Start take part as
// they are; StartStream flags its jobs (TAD_FLAG_SHARE) while sharing is on.  It takes effect for jobs that start after
// the call.  The controller calls it next to SetMemoryBudget.
func (r *gpuJobRunner) SetFitSharing(reserve uint64) error {
	if rc := C.tad_set_fit_sharing(r.ctx, C.uint64_t(reserve)); rc != C.TAD_OK {
		return fmt.Errorf("tad_set_fit_sharing: %s", C.GoString(C.tad_strerror(rc)))
	}
	r.share.Store(reserve != 0)
	return nil
}

// SetFitBeside lets an ARIMA job from Start fit beside another ARIMA job's fit while fit sharing is on (off by default):
// Start flags its ARIMA jobs (TAD_FLAG_FIT_BESIDE), and a flagged job queued behind a running fit then runs in that
// fit's reserve, its fit in one launch with the rest of the running one, instead of waiting for the whole fit phase.
// The running fit keeps about half the GPU meanwhile.  StartStream flags its ARIMA jobs too while fit sharing is on
// (SetFitSharing): a streamed job then fits beside a running fit once its SELECT has delivered its first block, and the
// running fit stays parked while further rounds of the SELECT are read.  It takes effect for jobs that start after the
// call.
func (r *gpuJobRunner) SetFitBeside(on bool) {
	r.beside.Store(on)
}

// SetStreamLend makes StartStream flag its jobs with TAD_FLAG_LEND (off by default).  While fit sharing is on
// (SetFitSharing), a streamed job then plans in the memory budget less the reserve and, while its worker waits for the
// SELECT's next block, runs the queued EWMA and DBSCAN jobs from Start in the reserve, so they no longer wait until the
// whole SELECT has been read; a block that arrives meanwhile waits for at most one such job.  It takes effect for jobs
// that start after the call.
func (r *gpuJobRunner) SetStreamLend(on bool) {
	r.lend.Store(on)
}

func algoCode(a string) C.int32_t {
	switch a {
	case "ARIMA":
		return C.TAD_ALGO_ARIMA
	case "DBSCAN":
		return C.TAD_ALGO_DBSCAN
	}
	return C.TAD_ALGO_EWMA
}

// fillColumn copies a Go slice into a library-owned pinned column, or -- for a key column the job does not use --
// zero-fills it (an all-zero column and a NULL column group identically).  tad_alloc_columns does not zero its
// buffers (cudaHostAlloc), so a short or missing slice must never leave part of a column unwritten: uninitialised
// bytes would be hashed into the connection key.
func fillColumn[T any](dst **T, src []T, n int, name string, required bool) error {
	if src == nil && !required {
		var zero T
		C.memset(unsafe.Pointer(*dst), 0, C.size_t(uintptr(n)*unsafe.Sizeof(zero)))
		return nil
	}
	if len(src) != n {
		return fmt.Errorf("column %s has %d values, flowEndSeconds has %d", name, len(src), n)
	}
	copy(unsafe.Slice(*dst, n), src)
	return nil
}

// Start replaces CreateSparkApplication (controller.go:685): non-blocking submit.
func (r *gpuJobRunner) Start(spec JobSpec, in *FlowColumns) error {
	n := len(in.FlowEnd)
	if spec.StartTime != 0 && in.FlowStart == nil {
		return illeagelArguementError{fmt.Errorf("invalid request: start_time needs the flow_start column")}
	}
	var cols C.tad_columns
	if rc := C.tad_alloc_columns(r.ctx, C.uint64_t(n), C.TAD_MEM_HOST, &cols); rc != C.TAD_OK {
		return fmt.Errorf("tad_alloc_columns: %s", C.GoString(C.tad_strerror(rc)))
	}
	fail := func(err error) error {
		C.tad_free_columns(r.ctx, &cols)
		return err
	}
	// library-owned pinned buffers: the engine never sees a Go pointer
	for _, err := range []error{
		fillColumn((**uint32)(unsafe.Pointer(&cols.src_ip)), in.SrcIP, n, "sourceIP", false),
		fillColumn((**uint32)(unsafe.Pointer(&cols.dst_ip)), in.DstIP, n, "destinationIP", false),
		fillColumn((**uint16)(unsafe.Pointer(&cols.src_port)), in.SrcPort, n, "sourceTransportPort", false),
		fillColumn((**uint16)(unsafe.Pointer(&cols.dst_port)), in.DstPort, n, "destinationTransportPort", false),
		fillColumn((**uint8)(unsafe.Pointer(&cols.proto)), in.Proto, n, "protocolIdentifier", false),
		fillColumn((**uint32)(unsafe.Pointer(&cols.flow_start)), in.FlowStart, n, "flowStartSeconds", false),
		fillColumn((**uint32)(unsafe.Pointer(&cols.flow_end)), in.FlowEnd, n, "flowEndSeconds", true),
		fillColumn((**uint64)(unsafe.Pointer(&cols.value)), in.Throughput, n, "throughput", true),
	} {
		if err != nil {
			return fail(err)
		}
	}
	cols.rows = C.uint64_t(n)

	js := C.tad_job_spec{algo: algoCode(spec.Algo), start_time: C.uint32_t(spec.StartTime), end_time: C.uint32_t(spec.EndTime),
		global_rows: C.uint64_t(spec.GlobalRows)}
	if spec.SumReducer {
		js.reducer = C.TAD_REDUCE_SUM
	}
	if len(spec.NSIgnore) > 0 {
		// namespace filter of the per-connection query (anomaly_detection.py:576-580): ids ride in two extra columns
		if rc := C.tad_alloc_ns_columns(r.ctx, &cols); rc != C.TAD_OK {
			return fail(fmt.Errorf("tad_alloc_ns_columns: %s", C.GoString(C.tad_strerror(rc))))
		}
		if err := fillColumn((**uint32)(unsafe.Pointer(&cols.src_ns)), in.SrcNS, n, "sourcePodNamespace", true); err != nil {
			return fail(err)
		}
		if err := fillColumn((**uint32)(unsafe.Pointer(&cols.dst_ns)), in.DstNS, n, "destinationPodNamespace", true); err != nil {
			return fail(err)
		}
		// tad_submit copies the list: the Go slice need not outlive the call (cgo pins it for its duration)
		js.n_ns_ignore = C.uint32_t(len(spec.NSIgnore))
		js.ns_ignore = (*C.uint32_t)(unsafe.Pointer(&spec.NSIgnore[0]))
	}
	if r.beside.Load() && js.algo == C.TAD_ALGO_ARIMA {
		js.flags |= C.TAD_FLAG_FIT_BESIDE
	}
	cid := C.CString(spec.ID)
	C.strncpy(&js.id[0], cid, 39)
	C.free(unsafe.Pointer(cid))

	var job *C.tad_job
	if rc := C.tad_submit(r.ctx, &js, &cols, &job); rc != C.TAD_OK {
		var st C.tad_status
		C.tad_poll(job, &st)
		msg := C.GoString(&st.err_msg[0])
		C.tad_release(job)
		C.tad_free_columns(r.ctx, &cols)
		return illeagelArguementError{fmt.Errorf("%s", msg)} // terminal FAILED, not retried (controller.go:505-514)
	}
	r.jobs.Store(spec.ID, &gpuJob{job: job, cols: cols})
	return nil
}

// BlockReader runs the job's SELECT once and calls emit for every block clickhouse-go hands over (the columns of one
// block, same layout as FlowColumns).  StartStream calls it once per round: it must return the same rows every time
// (a closed time window), in any order and block sizes.
type BlockReader func(emit func(*FlowColumns) error) error

// StartStream is Start for a table that never has to be in host memory at once (DESIGN.md section 10, single GPU): the
// rows go to the engine block by block as the SELECT delivers them, through two library-owned pinned blocks filled
// alternately, so block k+1 is decoded while block k is copied.  rowsHint is the SELECT count() (0 = unknown).  When the
// engine needs another hash-range pass it asks for the rows again and the SELECT is re-run.  Blocks larger than
// blockRows are cut.  Blocking: it returns when the input is complete.  The job is registered when it is submitted, so
// State and Cancel reach it while its rows are still being read (Cancel makes the feeding call return); Results works
// once the input is complete.
func (r *gpuJobRunner) StartStream(spec JobSpec, rowsHint uint64, blockRows int, read BlockReader) error {
	if blockRows <= 0 {
		return fmt.Errorf("blockRows must be positive")
	}
	var bufs [2]C.tad_columns
	freeBufs := func() {
		C.tad_free_columns(r.ctx, &bufs[0])
		C.tad_free_columns(r.ctx, &bufs[1])
	}
	for i := range bufs {
		if rc := C.tad_alloc_columns(r.ctx, C.uint64_t(blockRows), C.TAD_MEM_HOST, &bufs[i]); rc != C.TAD_OK {
			freeBufs()
			return fmt.Errorf("tad_alloc_columns: %s", C.GoString(C.tad_strerror(rc)))
		}
		if len(spec.NSIgnore) > 0 {
			if rc := C.tad_alloc_ns_columns(r.ctx, &bufs[i]); rc != C.TAD_OK {
				freeBufs()
				return fmt.Errorf("tad_alloc_ns_columns: %s", C.GoString(C.tad_strerror(rc)))
			}
		}
	}
	js := C.tad_job_spec{algo: algoCode(spec.Algo), start_time: C.uint32_t(spec.StartTime), end_time: C.uint32_t(spec.EndTime)}
	if spec.SumReducer {
		js.reducer = C.TAD_REDUCE_SUM
	}
	if r.share.Load() {
		// an ARIMA job's fit yields; an EWMA or DBSCAN job may run, its SELECT read, while a fit is parked
		js.flags |= C.TAD_FLAG_SHARE
		if r.beside.Load() && js.algo == C.TAD_ALGO_ARIMA {
			js.flags |= C.TAD_FLAG_FIT_BESIDE
		}
	}
	if r.lend.Load() {
		// the engine ignores the flag while fit sharing is off
		js.flags |= C.TAD_FLAG_LEND
	}
	// The ignore list goes as ids, and every block carries the SrcNS / DstNS ids the BlockReader's dictionary gave the
	// namespaces.  A reader that hands over the two namespace String columns as clickhouse-go received them (their
	// bytes and the offset of every 32nd row) would instead pass the list as names, in a tad_stream_filter_ns to
	// tad_submit_stream_filtered_ns with n_ns_ignore = 0 here, and each block's namespace text to
	// tad_stream_push_text_ns with src_ns / dst_ns NULL: the GPU then tests every row against the names and the host
	// builds no namespace dictionary (DESIGN.md section 10, "The namespace ignore list on the device").
	if len(spec.NSIgnore) > 0 {
		js.n_ns_ignore = C.uint32_t(len(spec.NSIgnore))
		js.ns_ignore = (*C.uint32_t)(unsafe.Pointer(&spec.NSIgnore[0]))
	}
	cid := C.CString(spec.ID)
	C.strncpy(&js.id[0], cid, 39)
	C.free(unsafe.Pointer(cid))
	var job *C.tad_job
	if rc := C.tad_submit_stream(r.ctx, &js, C.uint64_t(rowsHint), &job); rc != C.TAD_OK {
		var st C.tad_status
		C.tad_poll(job, &st)
		C.tad_release(job)
		freeBufs()
		return illeagelArguementError{fmt.Errorf("%s", C.GoString(&st.err_msg[0]))}
	}
	gj := &gpuJob{job: job, fed: make(chan struct{})}
	r.jobs.Store(spec.ID, gj)
	// engine errors: a bad block or a source that changed between rounds is terminal (controller.go:505-514)
	engineErr := func(call string, rc C.int) error {
		var st C.tad_status
		C.tad_poll(job, &st)
		err := fmt.Errorf("%s: %s: %s", call, C.GoString(C.tad_strerror(rc)), C.GoString(&st.err_msg[0]))
		if rc == C.TAD_ERR_INVALID_ARG {
			return illeagelArguementError{err}
		}
		return err
	}
	failed := func(err error) error {
		freeBufs() // push and end have returned: the engine no longer reads the blocks
		if _, mine := r.jobs.LoadAndDelete(spec.ID); mine {
			close(gj.fed)
			C.tad_release(job) // cancels a job whose input has not ended
		} else {
			close(gj.fed) // Cancel took the job and releases it
		}
		return err
	}
	k := 0
	push := func(in *FlowColumns, lo, n int) error {
		if spec.StartTime != 0 && in.FlowStart == nil {
			return illeagelArguementError{fmt.Errorf("invalid request: start_time needs the flow_start column")}
		}
		b := &bufs[k&1] // free again: the push of block k-1 has returned
		k++
		part := FlowColumns{}
		cut32 := func(s []uint32) []uint32 { if s == nil { return nil }; return s[lo : lo+n] }
		cut16 := func(s []uint16) []uint16 { if s == nil { return nil }; return s[lo : lo+n] }
		part.SrcIP, part.DstIP, part.FlowStart, part.FlowEnd = cut32(in.SrcIP), cut32(in.DstIP), cut32(in.FlowStart), cut32(in.FlowEnd)
		part.SrcPort, part.DstPort = cut16(in.SrcPort), cut16(in.DstPort)
		if in.Proto != nil {
			part.Proto = in.Proto[lo : lo+n]
		}
		part.Throughput = in.Throughput[lo : lo+n]
		for _, err := range []error{
			fillColumn((**uint32)(unsafe.Pointer(&b.src_ip)), part.SrcIP, n, "sourceIP", false),
			fillColumn((**uint32)(unsafe.Pointer(&b.dst_ip)), part.DstIP, n, "destinationIP", false),
			fillColumn((**uint16)(unsafe.Pointer(&b.src_port)), part.SrcPort, n, "sourceTransportPort", false),
			fillColumn((**uint16)(unsafe.Pointer(&b.dst_port)), part.DstPort, n, "destinationTransportPort", false),
			fillColumn((**uint8)(unsafe.Pointer(&b.proto)), part.Proto, n, "protocolIdentifier", false),
			fillColumn((**uint32)(unsafe.Pointer(&b.flow_start)), part.FlowStart, n, "flowStartSeconds", false),
			fillColumn((**uint32)(unsafe.Pointer(&b.flow_end)), part.FlowEnd, n, "flowEndSeconds", true),
			fillColumn((**uint64)(unsafe.Pointer(&b.value)), part.Throughput, n, "throughput", true),
		} {
			if err != nil {
				return err
			}
		}
		if len(spec.NSIgnore) > 0 {
			if err := fillColumn((**uint32)(unsafe.Pointer(&b.src_ns)), cut32(in.SrcNS), n, "sourcePodNamespace", true); err != nil {
				return err
			}
			if err := fillColumn((**uint32)(unsafe.Pointer(&b.dst_ns)), cut32(in.DstNS), n, "destinationPodNamespace", true); err != nil {
				return err
			}
		}
		b.rows = C.uint64_t(n)
		if rc := C.tad_stream_push(job, b); rc != C.TAD_OK {
			return engineErr("tad_stream_push", rc)
		}
		return nil
	}
	for again := C.int32_t(1); again != 0; {
		err := read(func(in *FlowColumns) error {
			for lo := 0; lo < len(in.FlowEnd); lo += blockRows {
				n := len(in.FlowEnd) - lo
				if n > blockRows {
					n = blockRows
				}
				if err := push(in, lo, n); err != nil {
					return err
				}
			}
			return nil
		})
		if err != nil {
			return failed(err)
		}
		if rc := C.tad_stream_end(job, &again); rc != C.TAD_OK {
			return failed(engineErr("tad_stream_end", rc))
		}
	}
	freeBufs() // the input is complete: the engine no longer reads the blocks
	close(gj.fed)
	return nil
}

// State replaces GetSparkApplication + the Spark-UI stage scraping (controller.go:426-497).
func (r *gpuJobRunner) State(id string) (state string, completed, total int, errMsg string) {
	v, ok := r.jobs.Load(id)
	if !ok {
		return "", 0, 0, "job not found"
	}
	var st C.tad_status
	C.tad_poll(v.(*gpuJob).job, &st)
	states := []string{"NEW", "SCHEDULED", "RUNNING", "COMPLETED", "FAILED"} // types.go:33-37
	return states[st.state], int(st.completed_stages), int(st.total_stages), C.GoString(&st.err_msg[0])
}

// Results hands every anomalous point to emit; the caller INSERTs into default.tadetector adding aggType /
// algoType / id / anomaly="true", or the "NO ANOMALY DETECTED" sentinel row when there is none
// (anomaly_detection.py:395-420).
func (r *gpuJobRunner) Results(id string, emit func(AnomalyRow)) (int, error) {
	v, ok := r.jobs.Load(id)
	if !ok {
		return 0, fmt.Errorf("job %s not found", id)
	}
	var rows C.tad_rows
	if rc := C.tad_result(v.(*gpuJob).job, &rows); rc != C.TAD_OK {
		return 0, fmt.Errorf("tad_result: %s", C.GoString(C.tad_strerror(rc)))
	}
	n := int(rows.rows)
	if n == 0 {
		return 0, nil
	}
	srcIP := unsafe.Slice((*uint32)(unsafe.Pointer(rows.src_ip)), n)
	dstIP := unsafe.Slice((*uint32)(unsafe.Pointer(rows.dst_ip)), n)
	srcPort := unsafe.Slice((*uint16)(unsafe.Pointer(rows.src_port)), n)
	dstPort := unsafe.Slice((*uint16)(unsafe.Pointer(rows.dst_port)), n)
	proto := unsafe.Slice((*uint8)(unsafe.Pointer(rows.proto)), n)
	fs := unsafe.Slice((*uint32)(unsafe.Pointer(rows.flow_start)), n)
	fe := unsafe.Slice((*uint32)(unsafe.Pointer(rows.flow_end)), n)
	sd := unsafe.Slice((*float64)(unsafe.Pointer(rows.stddev)), n)
	calc := unsafe.Slice((*float64)(unsafe.Pointer(rows.algo_calc)), n)
	thr := unsafe.Slice((*float64)(unsafe.Pointer(rows.throughput)), n)
	for i := 0; i < n; i++ {
		emit(AnomalyRow{srcIP[i], dstIP[i], fs[i], fe[i], srcPort[i], dstPort[i], proto[i], sd[i], calc[i], thr[i]})
	}
	return n, nil
}

// Cancel replaces DeleteSparkApplication (controller.go:385-424).
func (r *gpuJobRunner) Cancel(id string) {
	if v, ok := r.jobs.LoadAndDelete(id); ok {
		j := v.(*gpuJob)
		C.tad_cancel(j.job)
		if j.fed != nil {
			<-j.fed // a pending push or end returns TAD_ERR_CANCELLED; release only after the feeder has returned
		}
		C.tad_release(j.job)
		C.tad_free_columns(r.ctx, &j.cols)
	}
}

func (r *gpuJobRunner) Close() { C.tad_shutdown(r.ctx) }

// ipColumnFromNative turns the data part of a Native-format String column (sourceIP / destinationIP of a
// `SELECT ... FORMAT Native` block, create_table.sh:38-39) into the u32 key column.  isV4[i] == false marks rows
// whose text is not a dotted quad (IPv6, empty): the caller gives those dictionary ids.  Returns the number of
// bytes of buf the column occupied.
func ipColumnFromNative(buf []byte, rows int) (ips []uint32, isV4 []bool, used int, err error) {
	if rows == 0 || len(buf) == 0 {
		return nil, nil, 0, nil
	}
	offsets := make([]uint64, rows)
	lengths := make([]uint32, rows)
	var n C.size_t
	if rc := C.tad_ch_string_index((*C.uint8_t)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)), C.uint64_t(rows),
		(*C.uint64_t)(unsafe.Pointer(&offsets[0])), (*C.uint32_t)(unsafe.Pointer(&lengths[0])), &n); rc != C.TAD_OK {
		return nil, nil, 0, fmt.Errorf("malformed String column: %s", C.GoString(C.tad_strerror(rc)))
	}
	ips = make([]uint32, rows)
	flags := make([]uint8, rows)
	C.tad_ch_parse_ipv4((*C.uint8_t)(unsafe.Pointer(&buf[0])), (*C.uint64_t)(unsafe.Pointer(&offsets[0])),
		(*C.uint32_t)(unsafe.Pointer(&lengths[0])), C.uint64_t(rows), (*C.uint32_t)(unsafe.Pointer(&ips[0])),
		(*C.uint8_t)(unsafe.Pointer(&flags[0])))
	isV4 = make([]bool, rows)
	for i, f := range flags {
		isV4[i] = f != 0
	}
	return ips, isV4, int(n), nil
}
