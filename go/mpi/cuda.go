package mpi

// cuda.go -- the cgo shim: one Go method per C entry point of include/b200mpi.h.
// UNVERIFIED (no Go toolchain in the authoring image); see the package comment in mpi.go.
//
// Build: CGO_CFLAGS="-I<repo>/include" CGO_LDFLAGS="-L<repo>/mpi_b200/lib -lb200mpi" go build
//
// cgo rules observed here: Go pointers are handed to C only for the duration of one call and
// are never retained by the library (it stages or finishes before returning); empty slices pass
// a nil pointer (count 0 is legal in the ABI; bounce sends length-0 messages); blocking C calls
// occupy an OS thread, which is fine because every mpi call is blocking by contract.

/*
#cgo LDFLAGS: -lb200mpi
#include <stdlib.h>
#include "b200mpi.h"
*/
import "C"

import (
	"bytes"
	"encoding/gob"
	"errors"
	"fmt"
	"strings"
	"time"
	"unsafe"
)

// Cuda implements Interface and Collective on libb200mpi. Like Network in the reference, zero
// fields are filled from the -mpi-* flags at Init.
type Cuda struct {
	Addr     string        // address of the local process (-mpi-addr)
	Addrs    []string      // addresses of all processes (-mpi-alladdr)
	Timeout  time.Duration // Init fails after this long (-mpi-inittimeout); 0 waits forever
	Password string        // compared during the handshake (-mpi-password)
	Gpu      *int          // CUDA ordinal; nil takes -mpi-gpu (default -1: rank % device count)
}

const (
	dtU8  = C.B200MPI_U8
	dtI64 = C.B200MPI_I64
	dtF32 = C.B200MPI_F32
	dtF64 = C.B200MPI_F64
)

// DeviceSlice is device memory from the rank's peer-mapped heap; collectives and Send/Receive
// use it in place (no host staging).
type DeviceSlice struct {
	Ptr   unsafe.Pointer
	Len   int
	dtype C.int
	loc   bool // elements are value-location pairs of dtype values (AllreduceLoc and ReduceLoc only)
}

// Alloc returns a device slice of n elements shaped like the zero-length prototype, e.g.
// mpi.Alloc([]float32(nil), 1<<26), or mpi.Alloc([]Float64Loc(nil), n) for the pairs of AllreduceLoc.
func Alloc(prototype interface{}, n int) (*DeviceSlice, error) {
	var dt C.int
	var es int
	loc := false
	switch prototype.(type) {
	case []Float32Loc:
		dt, es, loc = dtF32, 16, true
	case []Float64Loc:
		dt, es, loc = dtF64, 16, true
	case []Int64Loc:
		dt, es, loc = dtI64, 16, true
	case []float32:
		dt, es = dtF32, 4
	case []float64:
		dt, es = dtF64, 8
	case []int64:
		dt, es = dtI64, 8
	case []byte:
		dt, es = dtU8, 1
	default:
		return nil, fmt.Errorf("mpi: no device slice of %T", prototype)
	}
	var p unsafe.Pointer
	if rc := C.b200mpi_alloc(C.size_t(n*es), &p); rc != 0 {
		return nil, lastError(rc, 0)
	}
	return &DeviceSlice{Ptr: p, Len: n, dtype: dt, loc: loc}, nil
}

// Free returns the slice to the heap.
func (d *DeviceSlice) Free() { C.b200mpi_free(d.Ptr); d.Ptr = nil }

// elemSize is the bytes of one element (16 for a value-location pair).
func (d *DeviceSlice) elemSize() int {
	switch {
	case d.loc:
		return 16
	case d.dtype == dtU8:
		return 1
	case d.dtype == dtF32:
		return 4
	}
	return 8
}

func lastError(rc C.int, tag int) error {
	msg := C.GoString(C.b200mpi_last_error())
	if rc == C.B200MPI_ERR_TAG_EXISTS {
		// the reference panics on a duplicate tag (network.go:469); surface it the same way
		panic(TagExists{Tag: tag}.Error())
	}
	return errors.New(msg)
}

func (c *Cuda) Init() error {
	if c.Password == "" {
		c.Password = FlagPassword
	}
	if c.Timeout == 0 {
		c.Timeout = time.Duration(FlagInitTimeout)
	}
	if c.Addr == "" {
		c.Addr = FlagAddr
	}
	if len(c.Addrs) == 0 {
		c.Addrs = append([]string(nil), FlagAllAddrs...)
	}
	gpu := FlagGpu
	if c.Gpu != nil {
		gpu = *c.Gpu
	}
	addr, all, pw := C.CString(c.Addr), C.CString(strings.Join(c.Addrs, ",")), C.CString(c.Password)
	defer C.free(unsafe.Pointer(addr))
	defer C.free(unsafe.Pointer(all))
	defer C.free(unsafe.Pointer(pw))
	if rc := C.b200mpi_init(addr, all, pw, C.int64_t(c.Timeout.Nanoseconds()), C.int(gpu)); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

func (c *Cuda) Finalize() { C.b200mpi_finalize() }
func (c *Cuda) Rank() int { return int(C.b200mpi_rank()) }
func (c *Cuda) Size() int { return int(C.b200mpi_size()) }

// lower turns `data interface{}` into (pointer, count, dtype, memkind). Anything that is not one
// of the typed slices is gob-encoded to bytes first, which keeps strings and structs working.
func lower(data interface{}) (unsafe.Pointer, int, C.int, C.int, error) {
	switch v := data.(type) {
	case *DeviceSlice:
		if v.loc {
			return nil, 0, 0, 0, errPairSlice
		}
		return v.Ptr, v.Len, v.dtype, C.B200MPI_DEVICE, nil
	case []float64:
		return ptr(len(v), func() unsafe.Pointer { return unsafe.Pointer(&v[0]) }), len(v), dtF64, C.B200MPI_HOST, nil
	case []float32:
		return ptr(len(v), func() unsafe.Pointer { return unsafe.Pointer(&v[0]) }), len(v), dtF32, C.B200MPI_HOST, nil
	case []int64:
		return ptr(len(v), func() unsafe.Pointer { return unsafe.Pointer(&v[0]) }), len(v), dtI64, C.B200MPI_HOST, nil
	case []byte:
		return ptr(len(v), func() unsafe.Pointer { return unsafe.Pointer(&v[0]) }), len(v), dtU8, C.B200MPI_HOST, nil
	case Raw:
		return ptr(len(v), func() unsafe.Pointer { return unsafe.Pointer(&v[0]) }), len(v), dtU8, C.B200MPI_HOST, nil
	}
	var buf bytes.Buffer
	if err := gob.NewEncoder(&buf).Encode(data); err != nil {
		return nil, 0, 0, 0, err
	}
	b := buf.Bytes()
	return ptr(len(b), func() unsafe.Pointer { return unsafe.Pointer(&b[0]) }), len(b), dtU8, C.B200MPI_HOST, nil
}

var errPairSlice = errors.New("mpi: a *DeviceSlice of value-location pairs goes through AllreduceLoc and ReduceLoc only")

func ptr(n int, f func() unsafe.Pointer) unsafe.Pointer {
	if n == 0 {
		return nil
	}
	return f()
}

func (c *Cuda) Send(data interface{}, destination, tag int) error {
	p, n, dt, kind, err := lower(data)
	if err != nil {
		return err
	}
	if rc := C.b200mpi_send(p, C.size_t(n), dt, C.int(destination), C.int(tag), kind); rc != 0 {
		return lastError(rc, tag)
	}
	return nil
}

// recvOnce is one b200mpi_recv call; n is the number of elements the message holds (also set
// when rc is B200MPI_ERR_TRUNCATE, in which case nothing was consumed and the call may be repeated
// with a larger buffer).
func recvOnce(p unsafe.Pointer, capacity int, dt, kind C.int, source, tag int) (n int, rc C.int) {
	var got C.size_t
	rc = C.b200mpi_recv(p, C.size_t(capacity), &got, dt, C.int(source), C.int(tag), kind)
	return int(got), rc
}

// recvBytes receives a byte message of unknown length into buf (grown when needed).
func recvBytes(buf []byte, source, tag int) ([]byte, error) {
	n, rc := recvOnce(ptr(len(buf), func() unsafe.Pointer { return unsafe.Pointer(&buf[0]) }), len(buf), dtU8, C.B200MPI_HOST, source, tag)
	if rc == C.B200MPI_ERR_TRUNCATE {
		buf = make([]byte, n)
		n, rc = recvOnce(unsafe.Pointer(&buf[0]), len(buf), dtU8, C.B200MPI_HOST, source, tag)
	}
	if rc != 0 {
		return nil, lastError(rc, tag)
	}
	return buf[:n], nil
}

// Receive takes a pointer to a slice (or a *DeviceSlice, or a pointer to any gob-decodable
// value). A slice that is too short is replaced by one of the sent length and the call repeated:
// the library keeps the message posted when it reports B200MPI_ERR_TRUNCATE. This is the
// resize-on-decode behaviour callers of the reference rely on (reference network.go:597).
func (c *Cuda) Receive(data interface{}, source, tag int) error {
	switch v := data.(type) {
	case *DeviceSlice:
		if v.loc {
			return errPairSlice
		}
		n, rc := recvOnce(v.Ptr, v.Len, v.dtype, C.B200MPI_DEVICE, source, tag)
		if rc != 0 {
			return lastError(rc, tag)
		}
		v.Len = n
		return nil
	case *[]float64:
		n, rc := recvOnce(ptr(len(*v), func() unsafe.Pointer { return unsafe.Pointer(&(*v)[0]) }), len(*v), dtF64, C.B200MPI_HOST, source, tag)
		if rc == C.B200MPI_ERR_TRUNCATE {
			*v = make([]float64, n)
			n, rc = recvOnce(unsafe.Pointer(&(*v)[0]), n, dtF64, C.B200MPI_HOST, source, tag)
		}
		if rc != 0 {
			return lastError(rc, tag)
		}
		*v = (*v)[:n]
		return nil
	case *[]float32:
		n, rc := recvOnce(ptr(len(*v), func() unsafe.Pointer { return unsafe.Pointer(&(*v)[0]) }), len(*v), dtF32, C.B200MPI_HOST, source, tag)
		if rc == C.B200MPI_ERR_TRUNCATE {
			*v = make([]float32, n)
			n, rc = recvOnce(unsafe.Pointer(&(*v)[0]), n, dtF32, C.B200MPI_HOST, source, tag)
		}
		if rc != 0 {
			return lastError(rc, tag)
		}
		*v = (*v)[:n]
		return nil
	case *[]int64:
		n, rc := recvOnce(ptr(len(*v), func() unsafe.Pointer { return unsafe.Pointer(&(*v)[0]) }), len(*v), dtI64, C.B200MPI_HOST, source, tag)
		if rc == C.B200MPI_ERR_TRUNCATE {
			*v = make([]int64, n)
			n, rc = recvOnce(unsafe.Pointer(&(*v)[0]), n, dtI64, C.B200MPI_HOST, source, tag)
		}
		if rc != 0 {
			return lastError(rc, tag)
		}
		*v = (*v)[:n]
		return nil
	case *[]byte:
		b, err := recvBytes(*v, source, tag)
		if err == nil {
			*v = b
		}
		return err
	case *Raw:
		b, err := recvBytes([]byte(*v), source, tag)
		if err == nil {
			*v = Raw(b)
		}
		return err
	}
	// anything else arrived gob-encoded (string, struct, ...): see lower()
	b, err := recvBytes(make([]byte, 256), source, tag)
	if err != nil {
		return err
	}
	return gob.NewDecoder(bytes.NewReader(b)).Decode(data)
}

// lowerTyped is lower() for the collectives: only typed slices, Raw and *DeviceSlice qualify. A
// gob-encoded temporary would receive the result instead of the caller's value (and its length
// may differ from rank to rank), so anything else is an error rather than a silent no-op.
func lowerTyped(what string, data interface{}) (unsafe.Pointer, int, C.int, C.int, error) {
	switch data.(type) {
	case *DeviceSlice, []float64, []float32, []int64, []byte, Raw:
		return lower(data)
	}
	return nil, 0, 0, 0, fmt.Errorf("mpi: %s needs []float64, []float32, []int64, []byte, Raw or *DeviceSlice, got %T", what, data)
}

func (c *Cuda) Bcast(data interface{}, root int) error {
	p, n, dt, kind, err := lowerTyped("Bcast", data)
	if err != nil {
		return err
	}
	if rc := C.b200mpi_bcast(p, C.size_t(n), dt, C.int(root), kind); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

func (c *Cuda) Allreduce(send, recv interface{}, op Op) error {
	sp, sn, sdt, sk, err := lowerTyped("Allreduce", send)
	if err != nil {
		return err
	}
	rp, rn, rdt, rk, err := lowerTyped("Allreduce", recv)
	if err != nil {
		return err
	}
	if sn != rn || sdt != rdt || sk != rk {
		return errors.New("mpi: Allreduce send and recv must have the same type, length and memory kind")
	}
	if rc := C.b200mpi_allreduce(sp, rp, C.size_t(sn), sdt, C.int(op), sk); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

func (c *Cuda) Allgather(send, recv interface{}) error {
	sp, sn, sdt, sk, err := lowerTyped("Allgather", send)
	if err != nil {
		return err
	}
	rp, rn, rdt, rk, err := lowerTyped("Allgather", recv)
	if err != nil {
		return err
	}
	if rn != sn*c.Size() || sdt != rdt || sk != rk {
		return errors.New("mpi: Allgather recv must hold Size()*len(send) elements of the same type")
	}
	if rc := C.b200mpi_allgather(sp, rp, C.size_t(sn), sdt, sk); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

// ReduceScatter: send holds Size() blocks of len(recv); rank j receives the reduction of block j.
func (c *Cuda) ReduceScatter(send, recv interface{}, op Op) error {
	sp, sn, sdt, sk, err := lowerTyped("ReduceScatter", send)
	if err != nil {
		return err
	}
	rp, rn, rdt, rk, err := lowerTyped("ReduceScatter", recv)
	if err != nil {
		return err
	}
	if sn != rn*c.Size() || sdt != rdt || sk != rk {
		return errors.New("mpi: ReduceScatter send must hold Size()*len(recv) elements of the same type")
	}
	if rc := C.b200mpi_reduce_scatter(sp, rp, C.size_t(rn), sdt, C.int(op), sk); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

// Reduce: Allreduce whose result lands on root only (recv may be nil elsewhere).
func (c *Cuda) Reduce(send, recv interface{}, op Op, root int) error {
	sp, sn, sdt, sk, err := lowerTyped("Reduce", send)
	if err != nil {
		return err
	}
	var rp unsafe.Pointer
	if recv != nil {
		var rn int
		var rdt, rk C.int
		rp, rn, rdt, rk, err = lowerTyped("Reduce", recv)
		if err != nil {
			return err
		}
		if sn != rn || sdt != rdt || sk != rk {
			return errors.New("mpi: Reduce send and recv must have the same type, length and memory kind")
		}
	}
	if rc := C.b200mpi_reduce(sp, rp, C.size_t(sn), sdt, C.int(op), C.int(root), sk); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

// scan lowers Scan and Exscan; Exscan's recv may be nil on rank 0, where it is not written.
func (c *Cuda) scan(what string, send, recv interface{}, op Op) error {
	sp, sn, sdt, sk, err := lowerTyped(what, send)
	if err != nil {
		return err
	}
	var rp unsafe.Pointer
	if recv != nil {
		var rn int
		var rdt, rk C.int
		rp, rn, rdt, rk, err = lowerTyped(what, recv)
		if err != nil {
			return err
		}
		if sn != rn || sdt != rdt || sk != rk {
			return fmt.Errorf("mpi: %s send and recv must have the same type, length and memory kind", what)
		}
	}
	var rc C.int
	if what == "Scan" {
		rc = C.b200mpi_scan(sp, rp, C.size_t(sn), sdt, C.int(op), sk)
	} else {
		rc = C.b200mpi_exscan(sp, rp, C.size_t(sn), sdt, C.int(op), sk)
	}
	if rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

// Scan: rank r's recv = send_0 op ... op send_r, combined in rank order.
func (c *Cuda) Scan(send, recv interface{}, op Op) error { return c.scan("Scan", send, recv, op) }

// Exscan: rank r's recv = send_0 op ... op send_{r-1}; rank 0's recv is not written.
func (c *Cuda) Exscan(send, recv interface{}, op Op) error { return c.scan("Exscan", send, recv, op) }

// Alltoall: block j of send becomes block Rank() of rank j's recv.
func (c *Cuda) Alltoall(send, recv interface{}) error {
	sp, sn, sdt, sk, err := lowerTyped("Alltoall", send)
	if err != nil {
		return err
	}
	rp, rn, rdt, rk, err := lowerTyped("Alltoall", recv)
	if err != nil {
		return err
	}
	if sn != rn || sn%c.Size() != 0 || sdt != rdt || sk != rk {
		return errors.New("mpi: Alltoall send and recv must both hold Size() equal blocks of the same type")
	}
	if rc := C.b200mpi_alltoall(sp, rp, C.size_t(sn/c.Size()), sdt, sk); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

// Isend is the Send of the design the reference sketches and comments out (mpi.go:132-143): it
// returns once data may be modified again, without waiting for the receiver.
func (c *Cuda) Isend(data interface{}, destination, tag int) error {
	p, n, dt, kind, err := lower(data)
	if err != nil {
		return err
	}
	if rc := C.b200mpi_isend(p, C.size_t(n), dt, C.int(destination), C.int(tag), kind); rc != 0 {
		return lastError(rc, tag)
	}
	return nil
}

// Wait blocks until destination confirmed the message sent with tag and frees the pair (mpi.go:146-152).
func (c *Cuda) Wait(destination, tag int) error {
	if rc := C.b200mpi_wait(C.int(destination), C.int(tag)); rc != 0 {
		return lastError(rc, tag)
	}
	return nil
}

// resized points the receiver at n elements: a slice behind a pointer is re-sliced when its array
// is large enough and replaced otherwise (as Receive does); a *DeviceSlice must hold n already.
func resized(what string, recv interface{}, n int) (interface{}, error) {
	switch v := recv.(type) {
	case *[]float64:
		if cap(*v) < n {
			*v = make([]float64, n)
		}
		*v = (*v)[:n]
		return *v, nil
	case *[]float32:
		if cap(*v) < n {
			*v = make([]float32, n)
		}
		*v = (*v)[:n]
		return *v, nil
	case *[]int64:
		if cap(*v) < n {
			*v = make([]int64, n)
		}
		*v = (*v)[:n]
		return *v, nil
	case *[]byte:
		if cap(*v) < n {
			*v = make([]byte, n)
		}
		*v = (*v)[:n]
		return *v, nil
	case *Raw:
		if cap(*v) < n {
			*v = make(Raw, n)
		}
		*v = (*v)[:n]
		return *v, nil
	case *DeviceSlice:
		if v.Len != n {
			return nil, fmt.Errorf("mpi: %s recv must hold %d elements", what, n)
		}
		return v, nil
	}
	return nil, fmt.Errorf("mpi: %s needs a pointer to []float64, []float32, []int64, []byte or Raw, or a *DeviceSlice, got %T", what, recv)
}

// lenOf is the element count of a recv passed as a pointer to a slice or as a *DeviceSlice.
func lenOf(recv interface{}) (int, bool) {
	switch v := recv.(type) {
	case *[]float64:
		return len(*v), true
	case *[]float32:
		return len(*v), true
	case *[]int64:
		return len(*v), true
	case *DeviceSlice:
		return v.Len, true
	}
	return 0, false
}

// table checks counts against Size() and returns it as the C array.
func (c *Cuda) table(what string, counts []int) ([]C.size_t, int, error) {
	if len(counts) != c.Size() {
		return nil, 0, fmt.Errorf("mpi: %s counts must hold Size() entries", what)
	}
	t := make([]C.size_t, len(counts))
	total := 0
	for i, n := range counts {
		if n < 0 {
			return nil, 0, fmt.Errorf("mpi: %s counts must not be negative", what)
		}
		t[i] = C.size_t(n)
		total += n
	}
	return t, total, nil
}

// lengths is every rank's element count, through one int64 Allgather.
func (c *Cuda) lengths(n int) ([]int, error) {
	all := make([]int64, c.Size())
	if err := c.Allgather([]int64{int64(n)}, all); err != nil {
		return nil, err
	}
	out := make([]int, len(all))
	for i, v := range all {
		out[i] = int(v)
	}
	return out, nil
}

func (c *Cuda) Gather(send, recv interface{}, root int) error {
	sp, sn, sdt, sk, err := lowerTyped("Gather", send)
	if err != nil {
		return err
	}
	var rp unsafe.Pointer
	if c.Rank() == root {
		r, err := resized("Gather", recv, sn*c.Size())
		if err != nil {
			return err
		}
		var rdt, rk C.int
		if rp, _, rdt, rk, err = lowerTyped("Gather", r); err != nil {
			return err
		}
		if sdt != rdt || sk != rk {
			return errors.New("mpi: Gather send and recv must have the same type and memory kind")
		}
	}
	if rc := C.b200mpi_gather(sp, rp, C.size_t(sn), sdt, C.int(root), sk); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

func (c *Cuda) Scatter(send, recv interface{}, root int) error {
	var sp unsafe.Pointer
	var sn int
	var sdt, sk C.int
	var err error
	r := recv
	if c.Rank() == root {
		if sp, sn, sdt, sk, err = lowerTyped("Scatter", send); err != nil {
			return err
		}
		if sn%c.Size() != 0 {
			return errors.New("mpi: Scatter send must hold Size() equal blocks")
		}
		if r, err = resized("Scatter", recv, sn/c.Size()); err != nil {
			return err
		}
	} else if r, err = resized("Scatter", recv, lenOf(recv)); err != nil {
		return err
	}
	rp, rn, rdt, rk, err := lowerTyped("Scatter", r)
	if err != nil {
		return err
	}
	if c.Rank() == root && (sdt != rdt || sk != rk) {
		return errors.New("mpi: Scatter send and recv must have the same type and memory kind")
	}
	if rc := C.b200mpi_scatter(sp, rp, C.size_t(rn), rdt, C.int(root), rk); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

// lenOf is the current length of the slice (or DeviceSlice) recv points to.
func lenOf(recv interface{}) int {
	switch v := recv.(type) {
	case *[]float64:
		return len(*v)
	case *[]float32:
		return len(*v)
	case *[]int64:
		return len(*v)
	case *[]byte:
		return len(*v)
	case *Raw:
		return len(*v)
	case *DeviceSlice:
		return v.Len
	}
	return 0
}

func (c *Cuda) gatherv(what string, send, recv interface{}, counts []int, root int, all bool) ([]int, error) {
	sp, sn, sdt, sk, err := lowerTyped(what, send)
	if err != nil {
		return nil, err
	}
	if counts == nil {
		if counts, err = c.lengths(sn); err != nil {
			return nil, err
		}
	}
	t, total, err := c.table(what, counts)
	if err != nil {
		return nil, err
	}
	if counts[c.Rank()] != sn {
		return nil, fmt.Errorf("mpi: %s counts[Rank()] must equal len(send)", what)
	}
	var rp unsafe.Pointer
	if all || c.Rank() == root {
		r, err := resized(what, recv, total)
		if err != nil {
			return nil, err
		}
		var rdt, rk C.int
		if rp, _, rdt, rk, err = lowerTyped(what, r); err != nil {
			return nil, err
		}
		if sdt != rdt || sk != rk {
			return nil, fmt.Errorf("mpi: %s send and recv must have the same type and memory kind", what)
		}
	}
	var rc C.int
	if all {
		rc = C.b200mpi_allgatherv(sp, rp, &t[0], sdt, sk)
	} else {
		rc = C.b200mpi_gatherv(sp, rp, &t[0], sdt, C.int(root), sk)
	}
	if rc != 0 {
		return nil, lastError(rc, 0)
	}
	return counts, nil
}

func (c *Cuda) Gatherv(send, recv interface{}, counts []int, root int) ([]int, error) {
	return c.gatherv("Gatherv", send, recv, counts, root, false)
}

func (c *Cuda) Allgatherv(send, recv interface{}, counts []int) ([]int, error) {
	return c.gatherv("Allgatherv", send, recv, counts, 0, true)
}

// ReduceScatterv: rank j's recv, resized to counts[j], receives op over every rank's block j in rank
// order. A nil counts on every rank is learnt from len(recv) with one Allgather. In place: recv points
// at this rank's block of send.
func (c *Cuda) ReduceScatterv(send, recv interface{}, counts []int, op Op) ([]int, error) {
	sp, sn, sdt, sk, err := lowerTyped("ReduceScatterv", send)
	if err != nil {
		return nil, err
	}
	if counts == nil {
		rn, ok := lenOf(recv)
		if !ok {
			return nil, fmt.Errorf("mpi: ReduceScatterv learns counts from a pointer to []float64, []float32 or []int64, or a *DeviceSlice, got %T", recv)
		}
		if counts, err = c.lengths(rn); err != nil {
			return nil, err
		}
	}
	t, total, err := c.table("ReduceScatterv", counts)
	if err != nil {
		return nil, err
	}
	if total != sn {
		return nil, errors.New("mpi: ReduceScatterv send must hold sum(counts) elements")
	}
	r, err := resized("ReduceScatterv", recv, counts[c.Rank()])
	if err != nil {
		return nil, err
	}
	rp, _, rdt, rk, err := lowerTyped("ReduceScatterv", r)
	if err != nil {
		return nil, err
	}
	if sdt != rdt || sk != rk {
		return nil, errors.New("mpi: ReduceScatterv send and recv must have the same type and memory kind")
	}
	if rc := C.b200mpi_reduce_scatterv(sp, rp, &t[0], sdt, C.int(op), sk); rc != 0 {
		return nil, lastError(rc, 0)
	}
	return counts, nil
}

// lowerLoc turns a pair slice (or a *DeviceSlice allocated with a pair prototype) into (pointer,
// pair count, dtype of the value, memkind). A nil slice is legal and lowers to a NULL pointer.
func lowerLoc(what string, data interface{}) (unsafe.Pointer, int, C.int, C.int, error) {
	switch v := data.(type) {
	case *DeviceSlice:
		if !v.loc {
			return nil, 0, 0, 0, fmt.Errorf("mpi: %s needs a *DeviceSlice of pairs (Alloc([]Float64Loc(nil), n))", what)
		}
		return v.Ptr, v.Len, v.dtype, C.B200MPI_DEVICE, nil
	case []Float32Loc:
		return ptr(len(v), func() unsafe.Pointer { return unsafe.Pointer(&v[0]) }), len(v), dtF32, C.B200MPI_HOST, nil
	case []Float64Loc:
		return ptr(len(v), func() unsafe.Pointer { return unsafe.Pointer(&v[0]) }), len(v), dtF64, C.B200MPI_HOST, nil
	case []Int64Loc:
		return ptr(len(v), func() unsafe.Pointer { return unsafe.Pointer(&v[0]) }), len(v), dtI64, C.B200MPI_HOST, nil
	}
	return nil, 0, 0, 0, fmt.Errorf("mpi: %s takes []Float32Loc, []Float64Loc, []Int64Loc or a *DeviceSlice of them, got %T", what, data)
}

// AllreduceLoc: MAXLOC (Max) / MINLOC (Min) over pairs, in rank order, into every rank's recv.
func (c *Cuda) AllreduceLoc(send, recv interface{}, op Op) error {
	sp, sn, sdt, sk, err := lowerLoc("AllreduceLoc", send)
	if err != nil {
		return err
	}
	rp, rn, rdt, rk, err := lowerLoc("AllreduceLoc", recv)
	if err != nil {
		return err
	}
	if sn != rn || sdt != rdt || sk != rk {
		return errors.New("mpi: AllreduceLoc send and recv must have the same length, pair type and memory kind")
	}
	if rc := C.b200mpi_allreduce_loc(sp, rp, C.size_t(sn), sdt, C.int(op), sk); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

// ReduceLoc: AllreduceLoc into root's recv only; recv may be nil elsewhere.
func (c *Cuda) ReduceLoc(send, recv interface{}, op Op, root int) error {
	sp, sn, sdt, sk, err := lowerLoc("ReduceLoc", send)
	if err != nil {
		return err
	}
	var rp unsafe.Pointer
	if recv != nil {
		var rn int
		var rdt, rk C.int
		if rp, rn, rdt, rk, err = lowerLoc("ReduceLoc", recv); err != nil {
			return err
		}
		if sn != rn || sdt != rdt || sk != rk {
			return errors.New("mpi: ReduceLoc send and recv must have the same length, pair type and memory kind")
		}
	}
	if rc := C.b200mpi_reduce_loc(sp, rp, C.size_t(sn), sdt, C.int(op), C.int(root), sk); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

// cudaWindow is a Window of libb200mpi: the id b200mpi_win_create handed out.
type cudaWindow struct{ id C.int }

// WinCreate: local's bytes (a pair slice too: a window is untyped memory), or an empty window for nil.
func (c *Cuda) WinCreate(local *DeviceSlice) (Window, error) {
	var base unsafe.Pointer
	var bytes C.size_t
	if local != nil {
		base, bytes = local.Ptr, C.size_t(local.Len*local.elemSize())
	}
	var id C.int
	if rc := C.b200mpi_win_create(base, bytes, &id); rc != 0 {
		return nil, lastError(rc, 0)
	}
	return &cudaWindow{id: id}, nil
}

// lowerOrigin is lowerTyped for the one-sided calls, which also refuse a negative displacement.
func lowerOrigin(what string, origin interface{}, disp int) (unsafe.Pointer, int, C.int, C.int, error) {
	if disp < 0 {
		return nil, 0, 0, 0, fmt.Errorf("mpi: %s displacement must be >= 0", what)
	}
	return lowerTyped(what, origin)
}

func (w *cudaWindow) Put(origin interface{}, target, disp int) error {
	p, n, dt, mk, err := lowerOrigin("Put", origin, disp)
	if err != nil {
		return err
	}
	if rc := C.b200mpi_put(p, C.size_t(n), dt, C.int(target), C.size_t(disp), w.id, mk); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

func (w *cudaWindow) Get(origin interface{}, target, disp int) error {
	p, n, dt, mk, err := lowerOrigin("Get", origin, disp)
	if err != nil {
		return err
	}
	if rc := C.b200mpi_get(p, C.size_t(n), dt, C.int(target), C.size_t(disp), w.id, mk); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

func (w *cudaWindow) Accumulate(origin interface{}, target, disp int, op Op) error {
	p, n, dt, mk, err := lowerOrigin("Accumulate", origin, disp)
	if err != nil {
		return err
	}
	if rc := C.b200mpi_accumulate(p, C.size_t(n), dt, C.int(op), C.int(target), C.size_t(disp), w.id, mk); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

func (w *cudaWindow) Fence() error {
	if rc := C.b200mpi_win_fence(w.id); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

func (w *cudaWindow) Free() error {
	if rc := C.b200mpi_win_free(w.id); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

// cudaWindow is also a PassiveWindow.
var _ PassiveWindow = (*cudaWindow)(nil)

func (w *cudaWindow) Lock(target int, lockType LockType) error {
	if lockType != LockExclusive && lockType != LockShared {
		return errors.New("mpi: lock type must be LockExclusive or LockShared")
	}
	if rc := C.b200mpi_win_lock(C.int(lockType), C.int(target), w.id); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

func (w *cudaWindow) Unlock(target int) error {
	if rc := C.b200mpi_win_unlock(C.int(target), w.id); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

// GetAccumulate: result must match origin's element type, length and memory kind (origin may be nil
// for NoOp).
func (w *cudaWindow) GetAccumulate(origin, result interface{}, target, disp int, op Op) error {
	rp, n, dt, mk, err := lowerOrigin("GetAccumulate", result, disp)
	if err != nil {
		return err
	}
	var optr unsafe.Pointer
	if origin != nil {
		p, on, odt, omk, err := lowerOrigin("GetAccumulate", origin, disp)
		if err != nil {
			return err
		}
		if on != n || odt != dt || omk != mk {
			return errors.New("mpi: GetAccumulate origin and result must have the same length, type and memory kind")
		}
		optr = p
	} else if op != NoOp {
		return errors.New("mpi: GetAccumulate needs an origin unless op is NoOp")
	}
	if rc := C.b200mpi_get_accumulate(optr, rp, C.size_t(n), dt, C.int(op), C.int(target), C.size_t(disp), w.id, mk); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

// FetchAndOp: value is a float32, float64 or int64 (an int is taken as int64); the previous value
// comes back with the same type. One kernel launch, no staging.
func (w *cudaWindow) FetchAndOp(value interface{}, target, disp int, op Op) (interface{}, error) {
	if disp < 0 {
		return nil, errors.New("mpi: FetchAndOp displacement must be >= 0")
	}
	if v, ok := value.(int); ok {
		value = int64(v)
	}
	var origin unsafe.Pointer
	var dt C.int
	var ret interface{}
	var result unsafe.Pointer
	switch v := value.(type) {
	case float32:
		r := new(float32)
		origin, dt, ret, result = unsafe.Pointer(&v), C.B200MPI_F32, r, unsafe.Pointer(r)
	case float64:
		r := new(float64)
		origin, dt, ret, result = unsafe.Pointer(&v), C.B200MPI_F64, r, unsafe.Pointer(r)
	case int64:
		r := new(int64)
		origin, dt, ret, result = unsafe.Pointer(&v), C.B200MPI_I64, r, unsafe.Pointer(r)
	default:
		return nil, fmt.Errorf("mpi: FetchAndOp takes a float32, float64 or int64, not %T", value)
	}
	if op == NoOp {
		origin = nil
	}
	if rc := C.b200mpi_fetch_and_op(origin, result, dt, C.int(op), C.int(target), C.size_t(disp), w.id); rc != 0 {
		return nil, lastError(rc, 0)
	}
	switch r := ret.(type) {
	case *float32:
		return *r, nil
	case *float64:
		return *r, nil
	default:
		return *(r.(*int64)), nil
	}
}

func (w *cudaWindow) CompareAndSwap(value, compare int64, target, disp int) (int64, error) {
	if disp < 0 {
		return 0, errors.New("mpi: CompareAndSwap displacement must be >= 0")
	}
	var old int64
	if rc := C.b200mpi_compare_and_swap(unsafe.Pointer(&value), unsafe.Pointer(&compare), unsafe.Pointer(&old), C.B200MPI_I64,
		C.int(target), C.size_t(disp), w.id); rc != 0 {
		return 0, lastError(rc, 0)
	}
	return old, nil
}

// cudaWindow is also a GroupWindow.
var _ GroupWindow = (*cudaWindow)(nil)

// cGroup: the ranks as a C int array (nil for an empty group); range and duplicates are the
// library's to check.
func cGroup(ranks []int) (*C.int, C.int) {
	if len(ranks) == 0 {
		return nil, 0
	}
	g := make([]C.int, len(ranks))
	for i, r := range ranks {
		g[i] = C.int(r)
		if int(g[i]) != r {
			g[i] = -1 // out of range either way
		}
	}
	return &g[0], C.int(len(g))
}

func (w *cudaWindow) Post(origins []int) error {
	p, n := cGroup(origins)
	if rc := C.b200mpi_win_post(p, n, w.id); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

func (w *cudaWindow) Start(targets []int) error {
	p, n := cGroup(targets)
	if rc := C.b200mpi_win_start(p, n, w.id); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

func (w *cudaWindow) Complete() error {
	if rc := C.b200mpi_win_complete(w.id); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

func (w *cudaWindow) Wait() error {
	if rc := C.b200mpi_win_wait(w.id); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}

func (w *cudaWindow) Test() (bool, error) {
	var flag C.int
	if rc := C.b200mpi_win_test(w.id, &flag); rc != 0 {
		return false, lastError(rc, 0)
	}
	return flag != 0, nil
}

// Scatterv: root always sends its table with one small Bcast, so the other ranks may pass nil.
func (c *Cuda) Scatterv(send, recv interface{}, counts []int, root int) ([]int, error) {
	n, isRoot := c.Size(), c.Rank() == root
	var sp unsafe.Pointer
	var sn int
	var sdt, sk C.int
	var err error
	if isRoot {
		if sp, sn, sdt, sk, err = lowerTyped("Scatterv", send); err != nil {
			return nil, err
		}
		if counts == nil {
			return nil, errors.New("mpi: Scatterv needs counts on root")
		}
	}
	if counts != nil {
		if _, total, err := c.table("Scatterv", counts); err != nil {
			return nil, err
		} else if isRoot && total != sn {
			return nil, errors.New("mpi: Scatterv send must hold sum(counts) elements on root")
		}
	}
	rootTable := make([]int64, n)
	if isRoot {
		for i, v := range counts {
			rootTable[i] = int64(v)
		}
	}
	if err := c.Bcast(rootTable, root); err != nil {
		return nil, err
	}
	if counts == nil { // a table that differs from root's fails as ERR_PEER on every rank
		counts = make([]int, n)
		for i, v := range rootTable {
			counts[i] = int(v)
		}
	}
	t, _, err := c.table("Scatterv", counts)
	if err != nil {
		return nil, err
	}
	r, err := resized("Scatterv", recv, counts[c.Rank()])
	if err != nil {
		return nil, err
	}
	rp, _, rdt, rk, err := lowerTyped("Scatterv", r)
	if err != nil {
		return nil, err
	}
	if isRoot && (sdt != rdt || sk != rk) {
		return nil, errors.New("mpi: Scatterv send and recv must have the same type and memory kind")
	}
	if rc := C.b200mpi_scatterv(sp, rp, &t[0], rdt, C.int(root), rk); rc != 0 {
		return nil, lastError(rc, 0)
	}
	return counts, nil
}

// Alltoallv: a nil recvCounts is learnt with one int64 Alltoall of sendCounts.
func (c *Cuda) Alltoallv(send interface{}, sendCounts []int, recv interface{}, recvCounts []int) ([]int, error) {
	sp, sn, sdt, sk, err := lowerTyped("Alltoallv", send)
	if err != nil {
		return nil, err
	}
	st, stotal, err := c.table("Alltoallv", sendCounts)
	if err != nil {
		return nil, err
	}
	if stotal != sn {
		return nil, errors.New("mpi: Alltoallv send must hold sum(sendCounts) elements")
	}
	if recvCounts == nil {
		mine, theirs := make([]int64, len(sendCounts)), make([]int64, len(sendCounts))
		for i, v := range sendCounts {
			mine[i] = int64(v)
		}
		if err := c.Alltoall(mine, theirs); err != nil {
			return nil, err
		}
		recvCounts = make([]int, len(theirs))
		for i, v := range theirs {
			recvCounts[i] = int(v)
		}
	}
	rt, rtotal, err := c.table("Alltoallv", recvCounts)
	if err != nil {
		return nil, err
	}
	r, err := resized("Alltoallv", recv, rtotal)
	if err != nil {
		return nil, err
	}
	rp, _, rdt, rk, err := lowerTyped("Alltoallv", r)
	if err != nil {
		return nil, err
	}
	if sdt != rdt || sk != rk {
		return nil, errors.New("mpi: Alltoallv send and recv must have the same type and memory kind")
	}
	if rc := C.b200mpi_alltoallv(sp, &st[0], rp, &rt[0], sdt, sk); rc != 0 {
		return nil, lastError(rc, 0)
	}
	return recvCounts, nil
}

func (c *Cuda) Barrier() error {
	if rc := C.b200mpi_barrier(); rc != 0 {
		return lastError(rc, 0)
	}
	return nil
}
